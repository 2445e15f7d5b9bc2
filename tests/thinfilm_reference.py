"""Extended-precision references of the thin-film and coating-design kernels (csrc/thinfilm.cu: pb_stack_eval,
pb_stack_grad, pb_field_at_depth, pb_coating_merit, pb_needle), numpy only.

Everything is evaluated in long double (`accuracy.LDBL`, complex `np.clongdouble`) from the exact fp64 values the device
received, following the maths of DESIGN §4.17 / §4.19 and the reference package's documented rules: the principal
square root of `_cos_snell` negated for a real sin theta > 1, numpy's signed zeros and complex division, the
multilayer_stack_rt assembly of r and t and the admittance assembly of the coatings engine.

Gradients are taken in forward mode, not by a reverse sweep: the tangent (dv_k / dp) of every layer thickness and the
real part of every layer index is carried through the substrate-to-ambient sweep next to v_k, from the closed forms of
dM_k / dbeta and dM_k / deta.  The needle function P(z) is the same tangent for the insertion of a needle layer of
thickness delta at z, dM / ddelta = M_top G M_bot.  Every seeded gradient is a linear functional of (R, T, A_k,
|E_k|^2) per sample, so one routine (`functional`) serves pb_stack_grad's four seeds, the six merit quantities and the
needle.  It returns each sample's contribution and a majorant (its terms with every product and real part taken in
absolute value, e.g. 2 |r| |dr| for dR = 2 Re(conj(r) dr)), so that a figure |g - g_ref| / majorant stays honest where
the sums over samples, boundaries or the real parts cancel.

The same code at complex128 (`model=True`) is a faithful fp64 model of the kernels; `defect=` plants one of the
regressions the GPU suite must catch (see DEFECTS).
"""
import numpy as np

from accuracy import LDBL, grid_for, sweep

PI_L = 4 * np.arctan(LDBL(1))
POL_S, POL_P, POL_AVG = 0, 1, 2
THINFILM, COATINGS = 0, 1
Q_R, Q_T, Q_ABS, Q_ESQ, Q_PEAK, Q_LAYER = range(6)
GRAD_TH, GRAD_IX = 1, 2

DEFECTS = {
    'beta32': 'beta (hence sin / cos beta) in float32',
    'stage32': 'a float32 field stage: v_k rounded to float32 before it is scaled by t',
    'esq_dropped': 'the 2 c_e E term of Ebar dropped',
    'ce_single': 'c_e not doubled',
    'seed_k': 'a field seed applied at boundary k instead of k + 1',
    'no_dcos': 'the index gradient without its dcos/dn term',
    'im_for_re': 'the index gradient taken for Im n instead of Re n',
    'slot_zero': 'the samples of one warp slot counted zero times',
    'slot_twice': 'the samples of one warp slot counted twice',
    'sweep2_overwrite': 'a warp slot overwritten on the second grid sweep instead of added to',
    'expm1_signed': 'e^{Im beta} formed as 1 + expm1(Im beta) with the sign kept',
    'peak_last': 'the peak seed sent to the last maximum rather than the first on a tie',
}


# ---- launch geometry (csrc/thinfilm.cu) ------------------------------------------------------------------------------
TF_THREADS = 256


def cm_threads(npol):
    """cm_threads: 128-thread blocks for the two-polarisation instances, 256 otherwise"""
    return 128 if npol == 2 else TF_THREADS


def warp_slots(count, sm_count, threads):
    """(W, nw): warp slots per partial row (grid_for blocks x threads / 32) and the slots tf_reduce sums"""
    W = grid_for(count, sm_count, threads) * threads // 32
    return W, min(W, (count + 31) // 32)


def visits(count, sm_count, threads):
    """grid sweeps of the warp-uniform loop: the most samples any warp slot takes, in passes of 32"""
    W, _ = warp_slots(count, sm_count, threads)
    return -(-count // (W * 32))


def cpad(count):
    """the stage pitch of the merit and needle kernels: count rounded up to whole warps"""
    return (count + 31) // 32 * 32


def straddle_counts(sm_count, threads):
    """warp edges, then one grid sweep - 1, exactly and + 1, and two sweeps + 33"""
    S = sweep(sm_count, threads)
    return (1, 31, 32, 33, S - 1, S, S + 1, 2 * S + 33)


def slot_sum(contrib, sm_count, threads, defect=None):
    """sum over samples (last axis) in fp64 through the kernel's warp slots: slot w holds the samples of passes
    base = 32 w + 32 W j; tf_reduce adds the first nw slots.  `defect` plants a slot fault (see DEFECTS)."""
    contrib = np.asarray(contrib, dtype=np.float64)
    count = contrib.shape[-1]
    W, nw = warp_slots(count, sm_count, threads)
    pad = -count % (32 * W)
    c = np.concatenate([contrib, np.zeros(contrib.shape[:-1] + (pad,))], axis=-1)
    per = c.reshape(contrib.shape[:-1] + (-1, W, 32)).sum(axis=-1)        # (..., passes, W)
    if defect == 'sweep2_overwrite':
        slots = per[..., -1, :] if per.shape[-2] > 1 else per[..., 0, :]
        if per.shape[-2] > 1:       # a slot the last pass missed keeps its earlier sum
            last = (count - 1 - 32 * np.arange(W) - 32 * W * (per.shape[-2] - 1)) >= 0
            slots = np.where(last, per[..., -1, :], per[..., -2, :])
    else:
        slots = per.sum(axis=-2)
        if defect == 'slot_zero':
            slots[..., 0] = 0.0
        elif defect == 'slot_twice':
            slots[..., 0] *= 2.0
    return slots[..., :nw].sum(axis=-1)


# ---- samples ---------------------------------------------------------------------------------------------------------
class Samples:
    """The six thin-film operands broadcast to their calculation shape and flattened: wvl, sin0 / cos0 (of the fp64
    product theta x theta_scale, as the device forms it), n0, nsub (P,), n, d (N, P).  `take(sl)` is a slice of the
    samples."""

    def __init__(self, wvl, theta, n0, nsub, n, d, theta_scale=1.0, model=False):
        self.model = model
        R, C = (np.float64, np.complex128) if model else (LDBL, np.clongdouble)
        n, d = np.asarray(n), np.asarray(d)
        N = max(n.shape[0], d.shape[0]) if n.ndim and d.ndim and min(n.shape[0], d.shape[0]) else 0
        calc = np.broadcast_shapes(*(np.shape(a) for a in (wvl, theta, n0, nsub)),
                                   *(a.shape[1:] for a in (n, d) if a.ndim))
        self.shape, self.N = calc, N
        P = int(np.prod(calc, dtype=np.int64))
        flat = lambda a, t: np.broadcast_to(np.asarray(a), calc).reshape(P).astype(t)
        self.wvl = flat(np.asarray(wvl, np.float64), R)
        th = np.broadcast_to(np.asarray(theta, np.float64), calc).reshape(P) * np.float64(theta_scale)
        self.sin0, self.cos0 = np.sin(th.astype(R)), np.cos(th.astype(R))
        self.n0 = flat(np.asarray(n0, np.complex128), C)
        self.nsub = flat(np.asarray(nsub, np.complex128), C)
        # a per-layer operand's calculation axes are right-aligned after its layer axis
        lay = lambda a, t: (np.broadcast_to(a.reshape(a.shape[:1] + (1,) * (len(calc) + 1 - a.ndim) + a.shape[1:]),
                                            (N,) + calc).reshape(N, P).astype(t) if N else np.zeros((0, P), t))
        self.n = lay(np.asarray(n, np.complex128), C)
        self.d = lay(np.asarray(d, np.float64), R)
        self.R, self.C = R, C
        self.pi = np.float64(np.pi) if model else PI_L

    def __len__(self):
        return self.wvl.shape[0]

    def take(self, sl):
        s = object.__new__(Samples)
        s.__dict__.update(self.__dict__)
        for k in ('wvl', 'sin0', 'cos0', 'n0', 'nsub'):
            setattr(s, k, getattr(self, k)[sl])
        s.n, s.d = self.n[:, sl], self.d[:, sl]
        return s


def chunks(S, size=1 << 16):
    for a in range(0, len(S), size):
        yield slice(a, min(a + size, len(S)))


# ---- complex helpers -------------------------------------------------------------------------------------------------
def cpx(re, im, C):
    """re + i im with signed zeros kept"""
    out = np.empty(np.broadcast(re, im).shape, C)
    out.real, out.imag = re, im
    return out


def cos_snell(n0, n, sin0, C):
    """_cos_snell: sqrt(1 - s^2) on the principal branch, s = (n0 / n) sin0 formed componentwise as the device does
    (so that the signed zero of Im s decides the branch), negated for a real s > 1"""
    q = n0 / n
    s = cpx(q.real * sin0 - q.imag * 0, q.real * 0 + q.imag * sin0, C)
    s2 = cpx(s.real * s.real - s.imag * s.imag, s.real * s.imag + s.imag * s.real, C)
    c = np.sqrt(cpx(1 - s2.real, 0 - s2.imag, C))
    flip = (s.imag == 0) & (s.real > 1)
    return np.where(flip, -c, c)


def admittance(n, cost, pol):
    return n / cost if pol == POL_P else n * cost


def sincos(beta, S, defect=None):
    """sin beta, cos beta of a complex beta: sin x cosh y + i cos x sinh y, cos x cosh y - i sin x sinh y"""
    x, y = beta.real, beta.imag
    if defect == 'expm1_signed':
        em1 = np.expm1(y)
        e = 1 + em1
        ch, sh = 0.5 * (e + 1 / e), 0.5 * em1 * (1 + 1 / e)
    else:
        ch, sh = np.cosh(y), np.sinh(y)
    sx, cx = np.sin(x), np.cos(x)
    return cpx(sx * ch, cx * sh, S.C), cpx(cx * ch, -sx * sh, S.C)


class Layer:
    """layer k of the samples: n, cos theta_k, beta, eta, sin / cos beta and dbeta/dd"""

    def __init__(self, S, k, pol, defect=None):
        self.n, self.d = S.n[k], S.d[k]
        self.cost = cos_snell(S.n0, self.n, S.sin0, S.C)
        self.dbdd = 2 * S.pi * self.n * self.cost / S.wvl
        self.beta = self.dbdd * self.d
        if defect == 'beta32':
            self.beta = self.beta.astype(np.complex64).astype(S.C)
        self.eta = admittance(self.n, self.cost, pol)
        self.sb, self.cb = sincos(self.beta, S, defect)


def apply(L_sb, L_cb, eta, v0, v1):
    """M v, M = [[cos b, -i sin b / eta], [-i eta sin b, cos b]]"""
    mis = -1j * L_sb
    return L_cb * v0 + mis / eta * v1, mis * eta * v0 + L_cb * v1


def substrate(S, pol, mode=COATINGS):
    """(v_N, eta_sub): [1, eta_sub], or multilayer_stack_rt's substrate column"""
    cs = cos_snell(S.n0, S.nsub, S.sin0, S.C)
    eta_sub = admittance(S.nsub, cs, pol)
    one = np.ones(len(S), S.C)
    if mode == THINFILM:
        return ((cs, S.nsub) if pol == POL_P else (one, S.nsub * cs)), eta_sub
    return (one, eta_sub), eta_sub


def eta0_of(S, pol):
    return admittance(S.n0, S.cos0.astype(S.C), pol)


# ---- forward sweep ---------------------------------------------------------------------------------------------------
def forward(S, pol, mode=COATINGS, defect=None):
    """dict of the forward outputs of one polarisation: r, t (P,); for COATINGS also v (N + 1, 2, P) unscaled, E, H,
    Esq (N + 1, P), R, T, A (N, P), eta0, eta_sub and the flux majorant Amaj of each A_k"""
    (v0, v1), eta_sub = substrate(S, pol, mode)
    N = S.N
    V = np.empty((N + 1, 2, len(S)), S.C)
    V[N] = v0, v1
    for k in range(N - 1, -1, -1):
        L = Layer(S, k, pol, defect)
        v0, v1 = apply(L.sb, L.cb, L.eta, v0, v1)
        V[k] = v0, v1
    out = {}
    if mode == THINFILM:
        term1 = 1 / (2 * S.n0 * S.cos0)
        a = S.n0 if pol == POL_P else S.n0 * S.cos0
        q1 = v1 * S.cos0 if pol == POL_P else v1
        A00, A10 = term1 * (a * v0 + q1), term1 * (a * v0 - q1)
        out['r'], out['t'] = A10 / A00, 1 / A00
        return out
    eta0 = eta0_of(S, pol)
    den = eta0 * v0 + v1
    r, t = (eta0 * v0 - v1) / den, 2 * eta0 / den
    t2 = (t * t.conj()).real
    Vs = V.astype(np.complex64).astype(S.C) if defect == 'stage32' else V
    g = (Vs[:, 0] * Vs[:, 1].conj()).real
    ga = np.abs(Vs[:, 0]) * np.abs(Vs[:, 1])         # the flux of a standing wave cancels: its majorant
    out.update(r=r, t=t, v=V, E=t * Vs[:, 0], H=t * Vs[:, 1], Esq=t2 * (Vs[:, 0] * Vs[:, 0].conj()).real,
               R=(r * r.conj()).real, T=eta_sub.real / eta0.real * t2, A=t2 * (g[:-1] - g[1:]) / eta0.real,
               Amaj=t2 * (ga[:-1] + ga[1:]) / np.abs(eta0.real), eta0=eta0, eta_sub=eta_sub)
    return out


# ---- tangents --------------------------------------------------------------------------------------------------------
def _layer_tangents(S, L, v0, v1, kinds, pol, N, k, defect=None):
    """{param: (dv0, dv1)} of dM_k / dp v_{k+1} for the parameters of layer k: thickness row k, index row N + k (the
    index rows follow the thickness rows only when both kinds are asked for)"""
    dM_db = lambda u0, u1: (-L.sb * u0 - 1j * L.cb / L.eta * u1, -1j * L.eta * L.cb * u0 - L.sb * u1)
    dM_de = lambda u0, u1: (1j * L.sb / (L.eta * L.eta) * u1, -1j * L.sb * u0)
    out = {}
    row = 0
    if kinds & GRAD_TH:
        a0, a1 = dM_db(v0, v1)
        out[k] = (L.dbdd * a0, L.dbdd * a1)
        row = N
    if kinds & GRAD_IX:
        n0s = S.n0 * S.sin0
        dcdn = n0s * n0s / (L.n ** 3 * L.cost)
        if defect == 'no_dcos':
            dcdn = dcdn * 0
        dbdn = 2 * S.pi * L.d / S.wvl * (L.cost + L.n * dcdn)
        dedn = 1 / L.cost - L.n * dcdn / (L.cost * L.cost) if pol == POL_P else L.cost + L.n * dcdn
        if defect == 'im_for_re':
            dbdn, dedn = 1j * dbdn, 1j * dedn
        a0, a1 = dM_db(v0, v1)
        b0, b1 = dM_de(v0, v1)
        out[row + k] = (dbdn * a0 + dedn * b0, dbdn * a1 + dedn * b1)
    return out


def functional(S, pol, coef, kinds=0, needle=None, defect=None):
    """The per-sample value of F = cR R + cT T + sum_k cA_k A_k + sum_k cE_k |E_k|^2 (coef = (cR, cT, cA, cE), any
    entry None; arrays over the samples, cA (N, P), cE (N + 1, P)) and, in forward mode, each sample's dF/dp and its
    majorant for the thickness / index parameters `kinds` asks for (rows as pb_stack_grad's output) or, with
    needle = (nn, zpart, layer of each depth), for the insertion of a needle layer at each depth.
    Returns (value, deriv (nparam, P), majorant (nparam, P))."""
    cR, cT, cA, cE = coef
    N, P = S.N, len(S)
    (v0, v1), eta_sub = substrate(S, pol)
    if needle is not None:
        nn, zpart, zl = needle
        cosn = cos_snell(S.n0, nn, S.sin0, S.C)
        eta_n = admittance(nn, cosn, pol)
        gdn = 2 * S.pi * nn * cosn / S.wvl
        npar = zpart.shape[1]
    else:
        npar = N * ((kinds & 1) + (kinds >> 1 & 1))
    D = np.zeros((npar, 2, P), S.C)
    z = np.zeros(P, S.R)
    zp = np.zeros((npar, P), S.R)
    Ev, Eva, Ed, Eda = z.copy(), z.copy(), zp.copy(), zp.copy()
    Av, Ava, Ad, Ada = z.copy(), z.copy(), zp.copy(), zp.copy()
    prev = None                      # (g, dg, v0, v1) of boundary k + 1

    def visit(k, v0, v1):
        nonlocal Ev, Eva, Av, Ava, prev, Ed, Eda, Ad, Ada
        g = (v0 * v1.conj()).real
        ga = np.abs(v0) * np.abs(v1)             # the flux of a standing wave cancels: its majorant
        dg = (D[:, 0] * v1.conj() + v0 * D[:, 1].conj()).real
        dga = np.abs(D[:, 0]) * np.abs(v1) + np.abs(v0) * np.abs(D[:, 1])
        if cE is not None:
            c = cE[k]
            if defect == 'esq_dropped':
                c = c * 0
            elif defect == 'ce_single':
                c = c * 0.5
            e2 = (v0 * v0.conj()).real
            Ev = Ev + cE[k] * e2
            Eva = Eva + np.abs(cE[k]) * e2
            if defect == 'seed_k' and prev is not None:
                de = 2 * (prev[2].conj() * D[:, 0]).real          # boundary k + 1's seed meets boundary k's tangent
                c = cE[k + 1]
            else:
                de = 2 * (v0.conj() * D[:, 0]).real
            Ed = Ed + c * de
            Eda = Eda + np.abs(c) * 2 * np.abs(v0) * np.abs(D[:, 0])
        if cA is not None and prev is not None:
            c = cA[k]
            Av = Av + c * (g - prev[0])
            Ava = Ava + np.abs(c) * (ga + prev[5])
            Ad = Ad + c * (dg - prev[1])
            Ada = Ada + np.abs(c) * (dga + prev[4])
        prev = (g, dg, v0, v1, dga, ga)

    visit(N, v0, v1)
    for k in range(N - 1, -1, -1):
        L = Layer(S, k, pol, None if defect == 'expm1_signed' else defect)
        if needle is not None:
            add = {}
            for j in np.nonzero(zl == k)[0]:
                # M_bot (the part of layer k below z), the generator G, then M_top
                sb, cb = sincos(L.dbdd * zpart[1, j], S)
                x0, x1 = apply(sb, cb, L.eta, v0, v1)
                x0, x1 = gdn * (-1j / eta_n) * x1, gdn * (-1j * eta_n) * x0
                sb, cb = sincos(L.dbdd * zpart[0, j], S)
                add[j] = apply(sb, cb, L.eta, x0, x1)
        else:
            add = _layer_tangents(S, L, v0, v1, kinds, pol, N, k, defect)
        D[:, 0], D[:, 1] = apply(L.sb, L.cb, L.eta, D[:, 0], D[:, 1])
        for p, (a0, a1) in add.items():
            D[p, 0] += a0
            D[p, 1] += a1
        v0, v1 = apply(L.sb, L.cb, L.eta, v0, v1)
        visit(k, v0, v1)
    eta0 = eta0_of(S, pol)
    den = eta0 * v0 + v1
    r, t = (eta0 * v0 - v1) / den, 2 * eta0 / den
    dden = eta0 * D[:, 0] + D[:, 1]
    dr = ((eta0 * D[:, 0] - D[:, 1]) - r * dden) / den
    dt = -t * dden / den
    t2 = (t * t.conj()).real
    dt2 = 2 * (t.conj() * dt).real
    # dr and dt cancel between the tangents of B and C: the majorant takes them apart
    ddena = (np.abs(eta0) * np.abs(D[:, 0]) + np.abs(D[:, 1])) / np.abs(den)
    dt2a = 2 * np.abs(t) * np.abs(t) * ddena
    kT = eta_sub.real / eta0.real
    val = t2 * Ev + t2 * Av / eta0.real
    der = dt2 * Ev + t2 * Ed + (dt2 * Av + t2 * Ad) / eta0.real
    maj = dt2a * Eva + t2 * Eda + (dt2a * Ava + t2 * Ada) / np.abs(eta0.real)
    if cR is not None:
        dR = 2 * (r.conj() * dr).real
        val, der = val + cR * (r * r.conj()).real, der + cR * dR
        maj = maj + np.abs(cR) * 2 * np.abs(r) * (1 + np.abs(r)) * ddena
    if cT is not None:
        val, der, maj = val + cT * kT * t2, der + cT * kT * dt2, maj + np.abs(cT * kT) * dt2a
    return val, der, maj


# ---- pb_stack_grad ---------------------------------------------------------------------------------------------------
def stack_grad(S, pol, kinds, seeds, defect=None):
    """(per-sample contributions (nparam, P), majorants (nparam, P)) of pb_stack_grad with seeds (dR, dT, dA, dEsq),
    any None, over the flattened samples; the output is contributions.sum(-1)."""
    der, maj = [], []
    for sl in chunks(S):
        c = tuple(None if s is None else s[..., sl] for s in seeds)
        _, d, m = functional(S.take(sl), pol, c, kinds, defect=defect)
        der.append(d)
        maj.append(m)
    return np.concatenate(der, -1), np.concatenate(maj, -1)


# ---- merit terms (pb_coating_merit) ----------------------------------------------------------------------------------
def _pols(pol):
    return (POL_S, POL_P) if pol == POL_AVG else (pol,)


def peak_arg(esq, blist, defect=None):
    """the list position of the first maximum of |E|^2 over the listed boundaries (NaN counts as the maximum)"""
    e = esq[list(blist)]
    if defect == 'peak_last':
        return len(blist) - 1 - np.argmax(e[::-1], axis=0)
    return np.argmax(e, axis=0)


def _coefs(S, quantity, b0, b1, blist, fwd, defect=None):
    """(value coefficients, gradient coefficients) of one polarisation's q as a functional of (R, T, A, |E|^2)"""
    N, P = S.N, len(S)
    one = np.ones(P, S.R)
    if quantity == Q_R:
        c = (one, None, None, None)
        return c, c
    if quantity == Q_T:
        c = (None, one, None, None)
        return c, c
    if quantity == Q_ABS:
        cA = np.zeros((N, P), S.R)
        cA[b0] = 1
        c = (None, None, cA, None)
        return c, c
    cE, gE = np.zeros((N + 1, P), S.R), np.zeros((N + 1, P), S.R)
    if quantity == Q_ESQ:
        cE[b0] = 1
        gE = cE
    elif quantity == Q_LAYER:
        cE[b0] += 0.5
        cE[b1] += 0.5
        gE = cE
    else:
        blist = list(blist)
        last = [all(blist[j] != blist[i] for j in range(i + 1, len(blist))) for i in range(len(blist))]
        arg = peak_arg(fwd['Esq'], blist, defect)
        idx = np.arange(P)
        cE[np.asarray(blist)[arg], idx] = 1
        keep = np.asarray(last)[arg]
        gE[np.asarray(blist)[arg], idx] = keep
    return (None, None, None, cE), (None, None, None, gE)


def merit(S, quantity, pol, target, weight, kinds=0, b0=0, b1=0, blist=None, defect=None, needle=None):
    """One merit term over the samples: dict of q (P,), resid = sqrt(w) (q - target) and its majorant rmaj =
    sqrt(w) (|q| + |target|), value terms w (q - target)^2 (P,)
    and, with kinds or needle = (nn, zpart, layer of each depth), the per-sample gradient contributions 2 w (q - target)
    / npol dq/dp and majorants (nparam, P)."""
    pols = _pols(pol)
    out = {k: [] for k in ('q', 'resid', 'rmaj', 'val', 'der', 'maj')}
    tg = np.broadcast_to(np.asarray(target, np.float64), S.shape).reshape(-1).astype(S.R)
    w = np.broadcast_to(np.asarray(weight, np.float64), S.shape).reshape(-1).astype(S.R)
    for sl in chunks(S):
        s = S.take(sl)
        q, parts = 0, []
        for p in pols:
            f = forward(s, p)
            vc, gc = _coefs(s, quantity, b0, b1, blist, f, defect)
            qp, d, m = functional(s, p, gc, kinds, needle=None if needle is None else (needle[0][sl],) + needle[1:],
                                  defect=defect) if (kinds or needle is not None) else (None, None, None)
            q = q + functional(s, p, vc)[0]
            parts.append((d, m))
        q = q / len(pols)
        dd = q - tg[sl]
        out['q'].append(q)
        out['resid'].append(np.sqrt(w[sl]) * dd)
        out['rmaj'].append(np.sqrt(w[sl]) * (np.abs(q) + np.abs(tg[sl])))
        out['val'].append(w[sl] * (dd * dd))
        if kinds or needle is not None:
            sc = 2 * w[sl] * dd / len(pols)
            out['der'].append(sum(sc * d for d, _ in parts))
            out['maj'].append(sum(np.abs(sc) * m for _, m in parts))
    return {k: np.concatenate(v, -1) for k, v in out.items() if v}


# ---- needle ----------------------------------------------------------------------------------------------------------
def depth_runs(Z, z, N):
    """the host's depth assignment of coatings._depth_runs: (zpart (2, nz), layer of each depth)"""
    j = np.clip(np.searchsorted(Z, z, side='right') - 1, 0, N - 1)
    return np.stack([z - Z[j], Z[j + 1] - z]).astype(np.float64), j


def needle(S, quantity, pol, target, weight, nn, zpart, zl, defect=None):
    """(per-sample contributions (nz, P), majorants) of P(z) for one R or T term; nn the needle index per sample"""
    nn = np.broadcast_to(np.asarray(nn, np.complex128), S.shape).reshape(-1).astype(S.C)
    m = merit(S, quantity, pol, target, weight, needle=(nn, zpart.astype(S.R), np.asarray(zl)), defect=defect)
    return m['der'], m['maj']


# ---- field at depth --------------------------------------------------------------------------------------------------
def field_at_depth(z, zb, n, n0, wvl, theta0, pol, Eb, Hb, model=False):
    """E, H at depths z from the boundary fields Eb, Hb (N + 1,): the layer of searchsorted(zb, z, 'right') - 1
    clipped to [0, N - 1], its part below z applied to the field at the layer's substrate-side boundary.  sin theta0
    is the host's fp64 sin, as pb_field_at_depth receives it."""
    R, C = (np.float64, np.complex128) if model else (LDBL, np.clongdouble)
    N = len(n)
    z = np.asarray(z, np.float64)
    li = np.clip(np.searchsorted(zb, z, side='right') - 1, 0, N - 1)
    S = object.__new__(Samples)
    S.R, S.C, S.pi = R, C, (np.float64(np.pi) if model else PI_L)
    nl = np.asarray(n, np.complex128)[li].astype(C)
    n0 = np.full(z.shape, complex(n0), C)
    sin0 = np.full(z.shape, np.sin(np.float64(theta0)), R)
    cost = cos_snell(n0, nl, sin0, C)
    eta = admittance(nl, cost, pol)
    beta = 2 * S.pi * nl * cost * (np.asarray(zb, np.float64)[li + 1].astype(R) - z.astype(R)) / R(wvl)
    sb, cb = sincos(beta, S)
    return apply(sb, cb, eta, np.asarray(Eb)[li + 1].astype(C), np.asarray(Hb)[li + 1].astype(C))


# ---- figures ---------------------------------------------------------------------------------------------------------
def rel_per_sample(got, ref):
    """max over samples of |got - ref| / |ref| (0 where both are 0)"""
    got, ref = np.asarray(got).astype(np.clongdouble), np.asarray(ref)
    den = np.abs(ref)
    e = np.abs(got - ref)
    with np.errstate(invalid='ignore', divide='ignore'):
        f = np.where(den > 0, e / np.where(den > 0, den, 1), np.where(e > 0, np.inf, 0))
    return float(np.max(f)) if f.size else 0.0


def rel_boundaries(got, ref):
    """fields (N + 1, P): max |got - ref| over each sample's largest boundary magnitude"""
    got, ref = np.asarray(got).astype(np.clongdouble), np.asarray(ref)
    den = np.abs(ref).max(axis=0)
    return float(np.max(np.abs(got - ref) / np.where(den > 0, den, 1))) if ref.size else 0.0


def over_majorant(got, ref, maj):
    """max |got - ref| / maj (a NaN or inf result stays one)"""
    got, ref, maj = (np.asarray(a) for a in (got, ref, maj))
    e = np.abs(got.astype(LDBL) - ref.astype(LDBL)) / np.where(maj > 0, maj, 1).astype(LDBL)
    e = np.where(np.isfinite(got), e, np.inf)
    return float(np.max(e)) if e.size else 0.0


def ulps32(got, ref, floor=None):
    """float32 outputs: max |got - ref| in ulps of the float32-rounded reference (of |ref| for a complex one), the ulp
    never below `floor` (a cancelling sum's fp64 majorant x 2^-52)"""
    got, ref = np.asarray(got), np.asarray(ref)
    sp = np.spacing(np.abs(ref).astype(np.float32)).astype(LDBL)
    if floor is not None:
        sp = np.maximum(sp, np.asarray(floor, LDBL) * LDBL(2.0 ** -52))
    e = np.abs(got.astype(np.clongdouble if np.iscomplexobj(got) else LDBL) - ref) / sp
    e = np.where(np.isfinite(got), e, np.inf)
    return float(np.max(e)) if e.size else 0.0
