"""Step-index fibers on the device (reference prysm/x/fibers.py): LP mode fields and mode coupling.

The mode fields come from one kernel, pb_lp_modes, which evaluates J_l with CUDA's fp64 Bessel functions and K_l with
its own exponentially scaled K (series / continued fraction for orders 0 and 1, upward recurrence above).  Coupling is
one fused reduction, pb_overlap: the field is read once per eight modes, everything accumulates in fp64, and the chunk
partials are summed in a fixed order, so the result is deterministic.

Couplings are 0-d device tensors (views of one (P,) tensor): nothing synchronises with the host until the caller asks,
and `float(eta)` gives the host value.

`find_all_modes` is host root-finding (scalar work); it brackets each root between its cutoff and the next pole and
solves the characteristic equation with scipy.
"""
import math

import numpy as np
import torch
from scipy import optimize, special

from . import _ops
from ._capi import LP_RULE_LP, LP_RULE_SMF, LP_NONE, LP_COS, LP_SIN
from .conf import config


def critical_angle(n_core, n_clad, deg=True):
    """Angle of total internal reflection in a step-index fiber (fibers.py:13-35)."""
    ang = np.arcsin(n_clad / n_core)
    return np.degrees(ang) if deg else ang


def numerical_aperture(n_core, n_clad):
    """NA of a step-index fiber (fibers.py:38-54)."""
    return np.sqrt(n_core * n_core - n_clad * n_clad)


def V(radius, NA, wavelength):
    """V number 2 pi / wavelength * radius * NA (fibers.py:57-83)."""
    return 2 * np.pi / wavelength * radius * NA


def marcuse_mfr_from_V(V):
    """Marcuse's mode field radius estimate w/a (fibers.py:462-479)."""
    return 0.65 + 1.619 * V ** -1.5 + 2.879 * V ** -6


def petermann_mfr_from_V(V):
    """Petermann's mode field radius estimate w/a (fibers.py:482-502)."""
    return marcuse_mfr_from_V(V) - 0.016 - 1.567 * V ** -7


# ---- mode finding (host) -------------------------------------------------------------------------------------------

def _bessel_zeros_below(order, limit):
    """Positive zeros of J_order below `limit`, ascending."""
    count = int(limit / np.pi) + 4
    while True:
        z = special.jn_zeros(order, count)
        if z[-1] >= limit:
            return z[z < limit]
        count *= 2


def _characteristic(U, V, l):
    """LHS - RHS of the LP characteristic equation in U (W = sqrt(V^2 - U^2)); zero at a guided mode.
    l = 0: U J1(U) / J0(U) = W K1(W) / K0(W);  l >= 1: U J_{l-1}(U) / J_l(U) = -W K_{l-1}(W) / K_l(W)."""
    W = math.sqrt(max(V * V - U * U, 0.0))
    if l == 0:
        return U * special.j1(U) / special.j0(U) - W * special.k1e(W) / special.k0e(W)
    return U * special.jv(l - 1, U) / special.jv(l, U) + W * special.kve(l - 1, W) / special.kve(l, W)


def _family(V, l):
    """(cutoffs, poles) in U of the LP_l family: LP_{0,m} starts at 0 and the zeros of J1, LP_{l,m} (l >= 1) at the
    zeros of J_{l-1}; the m-th root lies below the m-th zero of J_l (or below V)."""
    if l == 0:
        return np.concatenate(([0.0], _bessel_zeros_below(1, V))), _bessel_zeros_below(0, V)
    return _bessel_zeros_below(l - 1, V), _bessel_zeros_below(l, V)


def _solve_family(V, cutoffs, poles, l):
    eps = np.finfo(config.precision).eps
    roots = []
    for m, lo in enumerate(cutoffs):
        hi = min(poles[m] if m < len(poles) else V, V)
        if hi - lo <= 0:
            continue
        # stay off the cutoff and the pole, where the characteristic equation is 0/0 or infinite
        du = min(math.sqrt(eps) * max(V, 1.0), 1e-3 * (hi - lo))
        a, b = (lo + du if lo > 0 else du), hi - du
        if b <= a:
            continue
        fa, fb = _characteristic(a, V, l), _characteristic(b, V, l)
        while fa * fb > 0 and b - a > 4 * eps * V:    # a root hugging an end of the bracket: move the ends in
            du *= 1e-3
            a, b = (lo + du if lo > 0 else du), hi - du
            fa, fb = _characteristic(a, V, l), _characteristic(b, V, l)
        roots.append(optimize.brentq(_characteristic, a, b, args=(V, l), xtol=1e-15, rtol=4 * np.finfo(float).eps,
                                     maxiter=200))
    return np.asarray(roots, dtype=np.float64)


def find_all_modes(V, count_only=False):
    """Guided LP modes of a step-index fiber of V number V (fibers.py:289-340).

    Returns {l: b values} with keys 0, 1, -1, 2, -2, ... (the -l entries are the sine partners and share the b values
    of +l), or {l: number of modes} from cutoff theory when count_only.  As in the reference, the b values of a family
    are ascending: its lowest radial order, the largest b, comes last.
    """
    out = {}
    l = 0
    while True:
        cutoffs, poles = _family(V, l)
        if l > 0 and len(cutoffs) == 0:
            return out
        if count_only:
            out[l] = len(cutoffs)
            if l > 0:
                out[-l] = len(cutoffs)
        else:
            roots = _solve_family(V, cutoffs, poles, l)
            if len(roots):
                b = (1 - (roots / V) ** 2)[::-1].astype(config.precision)   # the reference's (ascending) order
                out[l] = b
                if l > 0:
                    out[-l] = b
        l += 1


# ---- mode fields (device) ------------------------------------------------------------------------------------------

def _real_grid(a):
    t = _ops.asdevice(a)
    if t.dtype != config.real_dtype:
        t = t.to(config.real_dtype)
    return t


def compute_LP_modes(V, mode_dict, a, r, t):
    """LP mode fields of a step-index fiber on the grids r, t (fibers.py:343-421), all from one pb_lp_modes launch.

    Returns {l: [field of each b]} with the structure of `mode_dict`.  The fields are views of one packed (P, *r.shape)
    device buffer, in mode_dict's key order and, within a key, in the reverse of its b order (the reference's
    `[::-1]`: descending b for find_all_modes' dicts, the lowest radial order first).  The core is
    r <= a; the cladding K_l(W r/a) / K_l(W); l > 0 carries cos(l t), l < 0 sin(|l| t).
    """
    r = _real_grid(r)
    t = _real_grid(t)
    plan, slots = [], []
    for l, bs in mode_dict.items():
        slots.append((l, len(bs)))
        az = LP_NONE if l == 0 else (LP_COS if l > 0 else LP_SIN)
        for b in np.asarray(bs, dtype=np.float64)[::-1]:
            plan.append((abs(l), abs(l), V * math.sqrt(1 - b), V * math.sqrt(b), LP_RULE_LP, az))
    packed = _ops.lp_modes(r, t, a, np.asarray(plan, dtype=np.float64).reshape(-1, 6))
    out, i = {}, 0
    for l, k in slots:
        out[l] = [packed[j] for j in range(i, i + k)]
        i += k
    return out


def smf_mode_field(V, a, b, r):
    """Mode field of a single-mode fiber (fibers.py:424-459): J0(U r/a) / J1(U) where r/a < 1, K0(W r/a) / K1(W)
    outside, with r/a formed as r * (1/a).  The reference's J1 / K1 denominators are kept, so the field is continuous at
    r = a only when U = W (b = 0.5)."""
    r = _real_grid(r)
    plan = np.array([[0, 1, V * math.sqrt(1 - b), V * math.sqrt(b), LP_RULE_SMF, LP_NONE]], dtype=np.float64)
    return _ops.lp_modes(r, None, a, plan)[0]


# ---- coupling ------------------------------------------------------------------------------------------------------

def _sum_arg(v):
    """An optional intensity sum as a (1,) fp64 device tensor (a host number is uploaded)."""
    if v is None:
        return None
    if isinstance(v, torch.Tensor):
        return v.detach().to(device=_ops.device() if not v.is_cuda else v.device, dtype=torch.float64).reshape(1)
    return torch.tensor([float(v)], dtype=torch.float64, device=_ops.device())


def _field_of(E, rdtype=None):
    E = _ops.asdevice(getattr(E, 'data', E))
    if rdtype is not None:
        E = E.to(_ops._CPLX_OF[rdtype] if E.is_complex() else rdtype)
    return E


def _coupling(E, modes, ip=None, ie=None, want_c=False):
    """pb_overlap with the field E (made complex) and the modes (real or complex, made E's precision)."""
    E = _field_of(E)
    if not E.is_complex():
        E = _ops.ascomplex(E)
    rd = _ops._REAL_OF[E.dtype]
    if isinstance(modes, torch.Tensor):
        modes = _field_of(modes, rd)
    else:
        modes = [_field_of(m, rd) for m in modes]
    return _ops.overlap(E, modes, ip=_sum_arg(ip), ie=_sum_arg(ie), want_c=want_c)


def mode_overlap_integral(E1, E2, E2conj=None, I1sum=None, I2sum=None):
    """eta = |sum E1 conj(E2)|^2 / (sum |E1|^2 sum |E2|^2) as a 0-d device tensor (fibers.py:505-548).

    One pb_overlap pass: E2 is conjugated on the fly, so E2conj is accepted for the reference's signature and not
    needed.  I1sum / I2sum (host numbers or device tensors) replace the corresponding sums.
    """
    eta, _ = _coupling(E2, [E1], ip=I1sum, ie=I2sum)
    return eta[0]


def _packed_base(ms):
    """The (P, ...) view of one buffer when the tensors ms are its consecutive planes (compute_LP_modes' output), else
    None."""
    m0 = ms[0]
    if not all(isinstance(m, torch.Tensor) and m.is_cuda and m.is_contiguous() for m in ms):
        return None
    n, es = m0.numel(), m0.element_size()
    for k, m in enumerate(ms):
        if (m.shape != m0.shape or m.dtype != m0.dtype or m.device != m0.device or
                m.untyped_storage().data_ptr() != m0.untyped_storage().data_ptr() or
                m.data_ptr() != m0.data_ptr() + k * n * es):
            return None
    return m0.as_strided((len(ms), *m0.shape), (n, *m0.stride()), m0.storage_offset())


def multimode_coupling(E_in, mode_fields):
    """Per-LP-mode coupling efficiency of the incident field E_in (fibers.py:551-588): {l: [eta of each mode]}.

    One pb_overlap for all modes: views of one packed buffer (compute_LP_modes) are read in place as that buffer, any
    other modes through a pointer list, never gathered.  The values are 0-d device tensors, views of one (P,) tensor.
    """
    keys = [(l, len(ms)) for l, ms in mode_fields.items()]
    flat = [m for ms in mode_fields.values() for m in ms]
    if not flat:
        return {l: [] for l, _ in keys}
    packed = _packed_base(flat)
    eta, _ = _coupling(E_in, packed if packed is not None else flat)
    out, i = {}, 0
    for l, k in keys:
        out[l] = [eta[j] for j in range(i, i + k)]
        i += k
    return out
