"""The GPU clients of the core kernels (DESIGN.md §1, "§8f") element by element against a high-precision reference.

Entry points and the kernels they run:
- `dspb200_conv_nd_exec(_dev)` with nffts (N-D :fft_simple), and `dspb200_conv_fft_exec` (1-D :fft_simple, its rank-1 case):
  `nd_copy_kernel`, `scale_cplx_kernel`, `os_cmul_kernel` + cuFFT;
- `dspb200_conv_nd_os_exec(_dev)` (N-D overlap-save): `nd_os_gather_kernel`, `nd_os_scatter_kernel` + batched cuFFT;
- `dspb200_hilbert_exec(_dev)`: `hilbert_weight_kernel` between a strided R2C and a batched C2C transform;
- `dspb200_periodogram2_exec(_dev)`: `per2_pad_kernel`, `per2_full_kernel`, `per2_radial_kernel`, `per2_radial_finish_kernel`;
- `dspb200_mt_cross_spectra_exec(_dev)`: `cs_prep_kernel`, `cs_acc_kernel`, `coherence_kernel` over the STFT kernels.

References are exact (int64 convolutions of integer data) or computed in high precision: float64 for Float32 kernels,
np.longdouble for Float64 kernels (direct sums, and numpy FFTs).  u is the eps of the real eltype, c = C_FFT = 2 (the constant
of tests/test_spectral_kernel_paths.py), and every bound is checked per element, so no large output can hide a small
broken one:
- convolution: |y - y_ref| <= c u log2(max(prod(nffts), 2)) ||u||_2 ||v||_2 (nffts: the block transform for overlap-save).
  Integer data is scaled so that this bound stays below 1/4: then rint(y) must equal the int64 convolution exactly.
- hilbert: |y - y_ref| <= c u log2(max(n, 2)) ||x_col||_2 / sqrt(n), and |Re y - x| within the same bound.
- 2-D periodogram, full form: the Welch bound of DESIGN.md §4 with m = 1, N = nfft1 nfft2 and E = sum s^2, plus u S for the
  rounding of 1/r to the signal type and 2 u log2(N) S for a bin dominated by the plane wave (the transform's error there
  is relative to the bin).  Radial forms: the sum of those bin bounds over a ring (times the ring weight 1 or 2)
  plus u |ring| for the final rounding; rings are restated from fft2pow2radial! with its exact expression
  round(Int, sqrt(muladd(a, a, kj2))), the fused multiply-add emulated exactly.  The ring populations must match exactly.
- multitaper cross spectra: per entry sum_t c_f (|da_t||b_t| + |a_t||db_t| + |da_t||db_t| + (T + 1) u |a_t||b_t|) with T
  tapers (one rounding per product and per running sum), |da_t| <= c u log2(nfft) ||x_l w_t||_2 (w_t the pre-scaled
  taper).  `demean` subtracts a mean rounded to the signal type, as the reference's `x .- mean(x)` does: that is a
  constant offset of up to u |mean_l|, so |da_t| gets u |mean_l| ||w_t||_1 more.  The same bound covers |Im S_ll| (the
  kernel's contracted a*conj(b) leaves a rounding-sized imaginary part on the diagonal, and S_lm and conj(S_ml) may differ
  in the last bit).  Coherence is checked against the interval the S bounds allow.

Calibration on an H100 80GB HBM3 (700 W).  Convolutions and multitaper cross spectra hold c = 2 with room to spare (largest
ratios 0.34 and 0.51).  Hilbert and the 2-D periodogram run cuFFT alone, and at c = 2 cuFFT missed: a plane wave's spur
bins in a Float32 80 x 45 transform reached 1.48 times the bound, Hilbert at the Bluestein size n = 1031 (Float64) 1.1 times,
and the peak bin of a Float64 1031 x 31 periodogram was off by 4.3 u relative (5 ulps), an error relative to the bin that
the per-bin model above does not contain.  At c = 3 with that relative term, a spur of the plane wave in a Float64
2 x 4096 transform still reached 1.29 times the bound.  So Hilbert uses c = C_HILBERT = 3, and the periodogram c = C_PER2 = 5
with the relative term 2 u log2(N) S.  cuFFT's batched Bluestein transforms (n = 1031) also couple the columns of one call: a weak
column next to strong ones had errors of 0.8 to 1.7 u ||x_neighbour|| / sqrt(n), far above its own norm allows, while the
same sizes with three columns of equal scale, and every smooth or small odd n with 64 columns, stayed within the
per-column bound.  hilbert_weight_kernel works element by element inside one column, so at non-smooth n the Hilbert bound
takes the largest column norm of the call.  test_report_largest_ratio prints the ratios per family, eltype and size class
(non-smooth: a prime factor above 7).

The CPU tests show that a correct single-precision computation passes each bound and that planted defects fail it.
Device inputs sit between sentinel samples of magnitude 10^6, device outputs between NaN cells that must survive every
call, and host outputs are followed by NaN cells too.  Host- and device-pointer forms run the same kernels and plans and
must agree bit for bit, except the radial periodograms: their Float64 atomics add in a run-to-run order."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import windows as ow

F32, F64, C64, C128 = (np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))
DTYPES = (F32, F64, C64, C128)
REALS = (F32, F64)
C_FFT = 2.0
C_HILBERT = 3.0   # hilbert and the 2-D periodogram run cuFFT alone: constants measured on the H100 (module docstring)
C_PER2 = 5.0
GUARD = 64
SENTINEL = 1e6
DEFAULT_BUDGET = 1 << 30          # g_nd_os_budget (overlap_save.cu)


def _cplx(dt):
    return np.dtype(dt).kind == "c"


def _f64(dt):
    return np.dtype(dt) in (F64, C128)


def _real(dt):
    return F64 if _f64(dt) else F32


def _ccx(dt):
    return C128 if _f64(dt) else C64


def eps(dt):
    return float(np.finfo(_real(dt)).eps)


def _hi(dt):
    """Reference precision: float64 for Float32 kernels, long double for Float64 kernels."""
    return np.longdouble if _f64(dt) else np.float64


def _hic(dt):
    return np.clongdouble if _f64(dt) else np.complex128


def cdiv(a, b):
    return -(-a // b)


def largest_prime(n):
    p, m, big = 2, n, 1
    while m > 1 and p * p <= m:
        while m % p == 0:
            big, m = p, m // p
        p += 1
    return max(big, m)


def nonsmooth(ns):
    """A transform size with a prime factor above 7 (cuFFT's Bluestein path)."""
    return any(largest_prime(int(n)) > 7 for n in ns)


def lg(n):
    return math.log2(max(int(n), 2))


# =============================================================================== N-D overlap-save geometry (restated)

def pad3(s):
    return tuple(s) + (1,) * (3 - len(s))


def os_geometry(dt, su, sv, nf, budget):
    """conv_nd_dev's ND_OS blocking (overlap_save.cu): L[d] = min(nf - sv + 1, so), nb[d] = ceil(so / L) and the blocks per
    batch, budget / per_block clamped to [1, nblocks]; per_block = one time-domain block + one spectrum (first dimension
    halved for real input).  Returns (so, L, nb, nblocks, batch)."""
    su, sv, nf = pad3(su), pad3(sv), pad3(nf)
    so = tuple(a + b - 1 for a, b in zip(su, sv))
    L = tuple(min(f - b + 1, o) for f, b, o in zip(nf, sv, so))
    nb = tuple(cdiv(o, l) for o, l in zip(so, L))
    nblocks = nb[0] * nb[1] * nb[2]
    batch = min(max(budget // os_per_block(dt, nf), 1), nblocks)
    return so, L, nb, nblocks, batch


def os_per_block(dt, nf):
    nf = pad3(nf)
    csz = 16 if _f64(dt) else 8
    nbins = (nf[0] if _cplx(dt) else nf[0] // 2 + 1) * nf[1] * nf[2]
    return nf[0] * nf[1] * nf[2] * np.dtype(dt).itemsize + nbins * csz


def os_budget(dt, su, sv, nf, regime):
    """The block-buffer budget that gives the batch regime: "one" block, a batch that "divides" the block count, one that
    does "not", or the default budget ("all" blocks in one batch)."""
    _, _, _, nblocks, _ = os_geometry(dt, su, sv, nf, DEFAULT_BUDGET)
    if regime == "all":
        return DEFAULT_BUDGET
    if regime == "one":
        b = 1
    elif regime == "divides":
        b = max(d for d in range(2, nblocks) if nblocks % d == 0)
    else:
        b = max(d for d in range(2, nblocks) if nblocks % d)
    return os_per_block(dt, nf) * b + os_per_block(dt, nf) // 2


def os_blocks(so, L, nb, nblocks, batch):
    """The scatter restated: per launch of nd_os_scatter_kernel (b0 = 0, batch, ...) every (block, j) it writes, as
    (block, j0, j1, j2, o0, o1, o2) rows."""
    rows = []
    for b0 in range(0, nblocks, batch):
        for lb in range(batch):
            b = b0 + lb
            if b >= nblocks:
                continue
            bb = (b % nb[0], (b // nb[0]) % nb[1], b // (nb[0] * nb[1]))
            j = np.stack(np.meshgrid(*[np.arange(l) for l in L], indexing="ij"), -1).reshape(-1, 3)
            o = j + np.asarray(L) * np.asarray(bb)
            keep = np.all(o < np.asarray(so), axis=1)
            rows.append(np.concatenate([np.full((keep.sum(), 1), b), j[keep], o[keep]], axis=1))
    return np.concatenate(rows)


# (su, sv, nf): rank 1-3, singleton dimensions, v larger than u along one dimension, a non-smooth block
OS_SHAPES = [
    ((1000,), (37,), (128,)),
    ((3000,), (100,), (1031,)),
    ((40, 30), (7, 45), (16, 64)),              # v longer than u along dimension 2
    ((1, 300), (1, 20), (1, 64)),
    ((12, 9, 10), (3, 4, 2), (8, 8, 4)),
    ((20, 1, 6), (5, 1, 3), (16, 1, 8)),
]
OS_REGIMES = ("one", "divides", "not", "all")


def os_cases(dt):
    """(su, sv, nf, regime) of test_conv_nd_os: every shape in the default regime, the multi-block shapes in all four."""
    cases = []
    for su, sv, nf in OS_SHAPES:
        nblocks = os_geometry(dt, su, sv, nf, DEFAULT_BUDGET)[3]
        regs = [r for r in OS_REGIMES if r == "all" or (r == "one" and nblocks > 1) or
                (r == "divides" and any(nblocks % d == 0 for d in range(2, nblocks))) or
                (r == "not" and any(nblocks % d for d in range(2, nblocks)))]
        cases += [(su, sv, nf, r) for r in regs]
    return cases


def test_restated_os_geometry():
    for dt in DTYPES:
        for su, sv, nf, regime in os_cases(dt):
            so, L, nb, nblocks, batch = os_geometry(dt, su, sv, nf, os_budget(dt, su, sv, nf, regime))
            want = {"one": lambda b: b == 1, "divides": lambda b: 1 < b < nblocks and nblocks % b == 0,
                    "not": lambda b: 1 < b < nblocks and nblocks % b, "all": lambda b: b == nblocks}[regime]
            assert want(batch), (dt, su, sv, nf, regime, batch, nblocks)
            rows = os_blocks(so, L, nb, nblocks, batch)
            # every output index is written by exactly one block
            count = np.zeros(so, dtype=np.int64)
            np.add.at(count, (rows[:, 4], rows[:, 5], rows[:, 6]), 1)
            assert (count == 1).all(), (su, sv, nf, regime)
            # output o = L b + j reads the block buffer at j + sv - 1 and needs the inputs o - (sv - 1) .. o, which lie at
            # j .. j + sv - 1 of the block's nf window (its first sample is u[L b - (sv - 1)])
            sv3, nf3 = np.asarray(pad3(sv)), np.asarray(pad3(nf))
            j = rows[:, 1:4]
            assert (j >= 0).all() and (j + sv3 - 1 < nf3).all()
            assert ((j + sv3 - 1) - (sv3 - 1) >= 0).all()
    # the table reaches every regime, every rank, singleton dimensions and v longer than u along one dimension
    regimes = {r for dt in DTYPES for *_, r in os_cases(dt)}
    assert regimes == set(OS_REGIMES)
    assert {len(su) for su, _, _ in OS_SHAPES} == {1, 2, 3}
    assert any(1 in su for su, _, _ in OS_SHAPES)
    assert any(any(b > a for a, b in zip(su, sv)) for su, sv, _ in OS_SHAPES)
    assert any(nonsmooth(nf) for _, _, nf in OS_SHAPES)
    assert os_geometry(F32, (1000,), (37,), (128,), DEFAULT_BUDGET)[1:4] == ((92, 1, 1), (12, 1, 1), 12)


# =============================================================================== references and bounds

def int_conv(u, v):
    """Exact convolution of integer arrays (complex: four int64 convolutions)."""
    from scipy.signal import convolve
    if np.iscomplexobj(u):
        ur, ui = u.real.astype(np.int64), u.imag.astype(np.int64)
        vr, vi = v.real.astype(np.int64), v.imag.astype(np.int64)
        cv = lambda a, b: convolve(a, b, method="direct")
        return cv(ur, vr) - cv(ui, vi) + 1j * (cv(ur, vi) + cv(ui, vr))
    return convolve(u.astype(np.int64), v.astype(np.int64), method="direct")


def hi_conv(u, v, dt):
    from scipy.signal import convolve
    h = _hic(dt) if _cplx(dt) else _hi(dt)
    return convolve(u.astype(h), v.astype(h), method="direct")


def conv_bound(u, v, nf, dt):
    n = float(np.prod(nf))
    return C_FFT * eps(dt) * lg(n) * float(np.linalg.norm(u.astype(np.complex128))) * float(np.linalg.norm(v.astype(np.complex128)))


def check_elems(y, ref, bound, what=""):
    """|y - ref| <= bound element by element (NaN fails); returns the largest error-to-bound ratio."""
    err = np.abs(np.asarray(y).astype(np.clongdouble) - np.asarray(ref).astype(np.clongdouble)).astype(np.float64)
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), err.shape)
    ok = err <= bound
    bad = np.argwhere(~ok)
    assert bad.size == 0, (what, bad[:6].tolist(), err[~ok][:4], bound[~ok][:4])
    return float(np.max(err / np.maximum(bound, 1e-300))) if err.size else 0.0


def conv_data(rng, shape, dt):
    g = rng.standard_normal(shape)
    if _cplx(dt):
        g = g + 1j * rng.standard_normal(shape)
    return g.astype(dt)


def int_pair(rng, su, sv, nf, dt):
    """Integer u, v drawn as large as keeps the convolution bound below 1/4, so that rint of a correct result is exact."""
    for amp in (64, 16, 4, 1):
        def draw(shape):
            g = rng.integers(-amp, amp + 1, shape).astype(np.float64)
            return (g + 1j * rng.integers(-amp, amp + 1, shape) if _cplx(dt) else g).astype(dt)
        u, v = draw(su), draw(sv)
        if conv_bound(u, v, nf, dt) < 0.25:
            return u, v
    raise AssertionError("no integer amplitude keeps the bound below 1/4")


def conv_pair(rng, su, sv, nf, dt, integer):
    return int_pair(rng, su, sv, nf, dt) if integer else (conv_data(rng, su, dt), conv_data(rng, sv, dt))


def hilbert_ref(x, dt):
    """Analytic signal of the columns of x (n x ncols) in high precision: bins 1 .. ceil(n/2) - 1 doubled, the negative
    half zeroed, DC and (n even) Nyquist kept."""
    n = x.shape[0]
    X = np.fft.fft(x.astype(_hi(dt)), axis=0)
    w = np.zeros(n)
    w[0] = 1
    w[1:(n + 1) // 2] = 2
    if n % 2 == 0:
        w[n // 2] = 1
    return np.fft.ifft(X * w[:, None].astype(_hi(dt)), axis=0)


def hilbert_bound(x, dt):
    """c u log2(n) ||x_col|| / sqrt(n) with c = C_HILBERT; at non-smooth n the largest column norm of the call (cuFFT's
    batched Bluestein transforms couple columns)."""
    n = x.shape[0]
    nrm = np.linalg.norm(x.astype(np.float64), axis=0)[None, :]
    if nonsmooth([n]):
        nrm = np.full_like(nrm, nrm.max())
    return C_HILBERT * eps(dt) * lg(n) * nrm / math.sqrt(n)


def power_bound(S, E, u, N, m, c=C_PER2):
    """DESIGN.md §4: the error of |X|^2 for an FFT accurate to c u log2(N) sqrt(E) per bin, plus m roundings of S, plus
    2 u log2(N) S: at a bin dominated by one tone the transform's error is relative to that bin, up to u per radix pass."""
    cu = c * u * lg(N)
    return 2 * cu * np.sqrt(S * E) + cu * cu * E + (m + 2 * lg(N)) * u * S


def per2_ref(s, f1, f2, dt):
    """|X|^2 of the zero-padded matrix (f1 x f2, high precision) and the signal energy."""
    pad = np.zeros((f1, f2), dtype=_hi(dt))
    pad[:s.shape[0], :s.shape[1]] = s
    X = np.fft.fft(np.fft.fft(pad, axis=0), axis=1)
    return (X.real ** 2 + X.imag ** 2).astype(np.float64), float(np.sum(s.astype(np.float64) ** 2))


def _fma_sqrt_rint(a, kj2):
    """rint(sqrt(fma(a, a, kj2))) elementwise, the fused multiply-add emulated exactly where it can change the ring."""
    t = a * a + kj2
    q = np.sqrt(t)
    w = np.rint(q)
    near = np.abs(q - np.floor(q) - 0.5) < 1e-6
    for idx in zip(*np.nonzero(near)):
        ex = float(Fraction(float(a[idx])) ** 2 + Fraction(float(kj2[idx])))      # correctly rounded: one rounding
        w[idx] = np.rint(math.sqrt(ex))
    return w.astype(np.int64)


def radial_rings(f1, f2, swap=False):
    """fft2pow2radial! (0-based): the ring of every half-spectrum bin (h x f2), its weight (1 on the row i = 0 and, f1
    even, the Nyquist row; 2 elsewhere) and kmax.  swap: c1 and c2 exchanged (a planted defect)."""
    h, nmin = f1 // 2 + 1, min(f1, f2)
    kmax = nmin // 2 + 1
    c1, c2 = (1.0, f1 / f2) if f1 == nmin else (f2 / f1, 1.0)
    if swap:
        c1, c2 = c2, c1
    i = np.arange(h, dtype=np.float64)[:, None] * np.ones((1, f2))
    j = np.arange(f2)[None, :] * np.ones((h, 1), dtype=np.int64)
    kj = np.where(j <= f2 // 2, j, j - f2).astype(np.float64) * c2
    ring = _fma_sqrt_rint(c1 * i, kj * kj)
    single = (i == 0) | ((i == h - 1) & (f1 % 2 == 0))
    return ring, np.where(single, 1, 2), kmax


def radial_ref(S, E, f1, f2, r, dt, rings=None):
    """Ring sums, ring bounds, populations and kmax of the radial forms from the full |X|^2 (f1 x f2)."""
    ring, mult, kmax = radial_rings(f1, f2) if rings is None else rings
    h = f1 // 2 + 1
    Sh = S[:h]
    bb = power_bound(Sh, E, eps(dt), f1 * f2, 2)
    keep = ring < kmax
    tot = np.zeros(kmax, dtype=np.longdouble)
    bnd = np.zeros(kmax)
    pop = np.zeros(kmax, dtype=np.int64)
    np.add.at(tot, ring[keep], (Sh.astype(np.longdouble) * mult / r)[keep])
    tot = tot.astype(np.float64)
    np.add.at(bnd, ring[keep], (bb * mult / r)[keep])
    np.add.at(pop, ring[keep], mult[keep])
    return tot, bnd + eps(dt) * tot, pop, kmax


def check_radial(sm, av, tot, bnd, pop, dt, what=""):
    """radialsum `sm` and radialavg `av` ring by ring, and the ring populations rint(sm / av) exactly."""
    r = check_elems(sm, tot, bnd, ("radialsum", what))
    r = max(r, check_elems(av, tot / pop, bnd / pop + eps(dt) * tot / pop, ("radialavg", what)))
    got = np.rint(sm.astype(np.float64) / av.astype(np.float64)).astype(np.int64)
    assert np.array_equal(got, pop), ("ring populations", what, got, pop)
    return r


def per2_signal(rng, n1, n2, dt):
    """A plane wave plus noise 10^-6 below it."""
    i = np.arange(n1)[:, None]
    j = np.arange(n2)[None, :]
    k1, k2 = n1 // 3, n2 // 5
    s = np.cos(2 * np.pi * (k1 * i / n1 + k2 * j / n2) + 0.3) + 1e-6 * rng.standard_normal((n1, n2))
    return s.astype(dt)


def mt_tapers(n, nt, weighted):
    """Taper rows w_t / sqrt(r_t) as MTConfig passes them: unit-norm dpss, r_t = 1 / weight_t (fs = 1), weights equal or
    the concentrations normalised to sum 1 (dpss_config's weight_by_evals)."""
    t = np.asarray(ow.dpss(n, 4, nt), dtype=np.float64).reshape(n, nt)
    t = t / np.sqrt(np.sum(t * t, axis=0, keepdims=True))
    if weighted:
        ev = np.asarray(ow.dpsseig(t, 4), dtype=np.float64)
        wts = ev / ev.sum()
    else:
        wts = np.full(nt, 1.0 / nt)
    return np.ascontiguousarray((t * np.sqrt(wts)[None, :]).T)


def mt_signal(rng, nchan, n, dt, offset):
    """nchan x n channels sharing a common tone (so that coherences spread over [0, 1]), plus a DC offset."""
    t = np.arange(n)
    common = np.sin(2 * np.pi * 0.1 * t)
    x = rng.standard_normal((nchan, n)) + common[None, :] * rng.uniform(0.2, 3, (nchan, 1)) + offset
    return x.astype(dt)


def mt_ref(x, rows, nfft, demean, dt):
    """Per taper spectra X (T x nchan x nout, high precision), c_f, and the per (taper, channel) bound on |dX|."""
    nchan, n = x.shape
    hi = _hi(dt)
    xh = x.astype(hi)
    mu = np.mean(x.astype(np.float64), axis=1) if demean else np.zeros(nchan)
    xd = xh - mu[:, None].astype(hi) if demean else xh
    nout = nfft // 2 + 1
    X = np.stack([np.fft.fft(xd * rows[t][None, :].astype(hi), nfft, axis=1)[:, :nout] for t in range(rows.shape[0])])
    cf = np.full(nout, 2.0)
    cf[0] = 1.0
    if nfft % 2 == 0:
        cf[-1] = 1.0
    u = eps(dt)
    xd64 = xd.astype(np.float64)
    dA = np.array([[C_FFT * u * math.log2(nfft) * np.linalg.norm(xd64[l] * rows[t]) +
                    (u * abs(mu[l]) * np.sum(np.abs(rows[t])) if demean else 0.0)
                    for l in range(nchan)] for t in range(rows.shape[0])])
    return X, cf, dA


def mt_cross_ref(X, cf, dA, f_lo, nf, dt):
    """S[l, m, fi] = sum_t c_f X_t[l, f] conj(X_t[m, f]) and its bound, f = f_lo + fi."""
    T = X.shape[0]
    Xs = X[:, :, f_lo:f_lo + nf]
    c = cf[f_lo:f_lo + nf]
    S = np.einsum("f,tlf,tmf->lmf", c.astype(Xs.real.dtype), Xs, np.conj(Xs))
    aX = np.abs(Xs).astype(np.float64)
    u = eps(dt)
    B = np.zeros(S.shape)
    for t in range(T):
        a, d = aX[t], dA[t]
        B += c[None, None, :] * (d[:, None, None] * a[None, :, :] + a[:, None, :] * d[None, :, None] +
                                 d[:, None, None] * d[None, :, None] + (T + 1) * u * a[:, None, :] * a[None, :, :])
    return S, B


def coherence_interval(S, B, dt):
    """The reference coherence and the interval [lo, hi] the bounds B of S allow (diagonal: 1)."""
    nchan = S.shape[0]
    d = np.real(np.stack([S[l, l] for l in range(nchan)])).astype(np.float64)
    db = np.stack([B[l, l] for l in range(nchan)])
    a = np.abs(S).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        ref = a / np.sqrt(d[:, None, :] * d[None, :, :])
        hi = (a + B) / np.sqrt(np.maximum(d - db, 0)[:, None, :] * np.maximum(d - db, 0)[None, :, :])
        lo = np.maximum(a - B, 0) / np.sqrt((d + db)[:, None, :] * (d + db)[None, :, :])
    hi = np.where(np.isnan(hi), np.inf, hi)
    u = eps(dt)
    hi, lo = hi * (1 + 4 * u), lo * (1 - 4 * u)
    for l in range(nchan):
        ref[l, l], hi[l, l], lo[l, l] = 1.0, 1.0, 1.0
    return ref, lo, hi


def check_coherence(Cg, ref, lo, hi, what=""):
    ok = (Cg >= lo) & (Cg <= hi) & (Cg >= 0)
    assert ok.all(), (what, np.argwhere(~ok)[:6].tolist())
    nchan = Cg.shape[0]
    for l in range(nchan):
        assert (Cg[l, l] == 1).all(), (what, "diagonal")
    assert (Cg <= np.maximum(1.0, hi)).all()
    half = np.where(Cg >= ref, hi - ref, ref - lo)
    err = np.abs(Cg - ref)
    return float(np.max(np.where(err > 0, err / np.maximum(half, 1e-300), 0.0)))


# =============================================================================== CPU: single-precision computations

def _sp_cfft(a, nf):
    return np.fft.fftn(a.astype(C64), nf, axes=tuple(range(len(nf))))


def sp_conv_fft(u, v, nf, dt):
    """A correct single-precision :fft_simple: complex64 transforms, V scaled by 1/prod(nf), unnormalised inverse."""
    U = _sp_cfft(u, nf)
    V = (_sp_cfft(v, nf) * np.float32(1.0 / np.prod(nf))).astype(C64)
    y = np.fft.ifftn((U * V).astype(C64), norm="forward").astype(C64)
    so = tuple(a + b - 1 for a, b in zip(u.shape, v.shape))
    y = y[tuple(slice(0, o) for o in so)]
    return y if _cplx(dt) else y.real.astype(F32)


def sp_conv_os(u, v, nf, dt, shift_block=None, halo=None):
    """A single-precision N-D overlap-save with the blocking of conv_nd_dev.  Planted defects: shift_block = one block
    whose outputs are read one sample early along dimension 1; halo = the block start taken `halo` samples before the
    block's first output instead of sv - 1."""
    rank = u.ndim
    su, sv, nf3 = pad3(u.shape), pad3(v.shape), pad3(nf)
    so, L, nb, nblocks, _ = os_geometry(F32, su, sv, nf3, DEFAULT_BUDGET)
    u3 = u.reshape(su).astype(C64)
    V = (np.fft.fftn(np.pad(v.reshape(sv).astype(C64), [(0, f - s) for f, s in zip(nf3, sv)])) *
         np.float32(1.0 / np.prod(nf3))).astype(C64)
    out = np.zeros(so, dtype=C64)
    for b in range(nblocks):
        bb = (b % nb[0], (b // nb[0]) % nb[1], b // (nb[0] * nb[1]))
        td = np.zeros(nf3, dtype=C64)
        start = [L[d] * bb[d] - ((sv[d] - 1) if halo is None or sv[d] == 1 else halo(sv[d])) for d in range(3)]
        src = [slice(max(s, 0), min(s + f, n)) for s, f, n in zip(start, nf3, su)]
        dst = [slice(sl.start - s, sl.stop - s) for sl, s in zip(src, start)]
        if all(sl.stop > sl.start for sl in src):
            td[tuple(dst)] = u3[tuple(src)]
        y = np.fft.ifftn((np.fft.fftn(td) * V).astype(C64), norm="forward").astype(C64)
        lo = [L[d] * bb[d] for d in range(3)]
        cnt = [min(L[d], so[d] - lo[d]) for d in range(3)]
        off = [sv[d] - 1 for d in range(3)]
        if shift_block == b:
            off[0] -= 1
        out[tuple(slice(l, l + c) for l, c in zip(lo, cnt))] = y[tuple(slice(o, o + c) for o, c in zip(off, cnt))]
    out = out.reshape(tuple(a + b - 1 for a, b in zip(u.shape, v.shape))) if rank < 3 else out
    return out if _cplx(dt) else out.real.astype(F32)


def sp_hilbert(x, defect=None):
    """A single-precision hilbert the way the kernels do it: rfft into the first n/2 + 1 bins, hilbert_weight_kernel's
    weights times 1/n, unnormalised inverse.  Planted defects: "nyquist doubled" (n even), "odd last not doubled" (n odd),
    "upper not zeroed" (the upper bins keep the mirror image a complex transform would leave there), "no 1/n"."""
    n = x.shape[0]
    full = np.fft.fft(x.astype(C64), axis=0).astype(C64)
    X = np.zeros_like(full)
    X[:n // 2 + 1] = np.fft.rfft(x.astype(F32), axis=0)
    w = np.ones(n)
    last2 = (n + 1) // 2 - 1
    w[1:last2 + 1] = 2
    w[n // 2 + 1:] = 0
    scale = 1.0 / n
    if defect == "nyquist doubled":
        w[n // 2] = 2
    elif defect == "odd last not doubled":
        w[last2] = 1
    elif defect == "upper not zeroed":
        X[n // 2 + 1:] = full[n // 2 + 1:]
        w[n // 2 + 1:] = 1
    elif defect == "no 1/n":
        scale = 1.0
    Xw = (X * (w * scale).astype(F32)[:, None]).astype(C64)
    return np.fft.ifft(Xw, axis=0, norm="forward").astype(C64)


def sp_per2_half(s, f1, f2):
    pad = np.zeros((f1, f2), dtype=F32)
    pad[:s.shape[0], :s.shape[1]] = s
    return np.fft.fft(np.fft.rfft(pad, axis=0).astype(C64), axis=1).astype(C64)


def sp_per2_full(s, f1, f2, r, defect=None):
    """per2_full_kernel in single precision; defect "mirror off by one": row n1 - 1 - i read for the mirrored rows."""
    Xh = sp_per2_half(s, f1, f2)
    h = f1 // 2 + 1
    i = np.arange(f1)[:, None]
    j = np.arange(f2)[None, :]
    mi = f1 - 1 - i if defect == "mirror off by one" else f1 - i
    src = np.where(i < h, Xh[np.minimum(i, h - 1), j], np.conj(Xh[np.clip(mi, 0, h - 1), (f2 - j) % f2]))
    p = (src.real * src.real + src.imag * src.imag).astype(F32)
    return (p * np.float32(1.0 / r)).astype(F32)


def sp_per2_radial(s, f1, f2, r, avg, defect=None):
    """per2_radial_kernel + finish in single precision (Float64 ring sums).  Defects: "nyquist row m2" (f1 even), "c1 c2
    swapped"."""
    Xh = sp_per2_half(s, f1, f2)
    ring, mult, kmax = radial_rings(f1, f2, swap=defect == "c1 c2 swapped")
    if defect == "nyquist row m2":
        mult = mult.copy()
        mult[-1] = 2
    m = np.where(mult == 1, float(np.float32(1.0 / r)), float(np.float32(2.0 / r)))
    p = (Xh.real * Xh.real + Xh.imag * Xh.imag).astype(F32).astype(np.float64)
    keep = ring < kmax
    acc = np.zeros(kmax)
    wc = np.zeros(kmax)
    np.add.at(acc, ring[keep], (p * m)[keep])
    np.add.at(wc, ring[keep], mult[keep])
    return (acc / wc if avg else acc).astype(F32)


def sp_mt_cross(x, rows, nfft, demean, f_lo, nf, defect=None):
    """cs_prep + STFT + cs_acc (+ coherence) in single precision.  Defects: "dc weight 2", "odd last weight 1",
    "f_lo ignored", "conj on a", "coherence upper stride"."""
    nchan, n = x.shape
    mu = np.mean(x.astype(np.float64), axis=1).astype(F32) if demean else np.zeros(nchan, F32)
    xd = (x - mu[:, None]).astype(F32)
    nout = nfft // 2 + 1
    S = np.zeros((nchan, nchan, nf), dtype=C64)
    for t in range(rows.shape[0]):
        seg = (xd.astype(np.float64) * rows[t][None, :]).astype(F32)
        X = np.fft.fft(seg.astype(C64), nfft, axis=1)[:, :nout].astype(C64)
        f = np.arange(nf) + (0 if defect == "f_lo ignored" else f_lo)
        c = np.where((f == 0) | ((nfft % 2 == 0) & (f == nout - 1)), 1.0, 2.0)
        if defect == "dc weight 2":
            c = np.where(f == 0, 2.0, c)
        if defect == "odd last weight 1":
            c = np.where(f == nout - 1, 1.0, c)
        a, b = X[:, None, f], X[None, :, f]
        v = (np.conj(a) * b if defect == "conj on a" else a * np.conj(b)).astype(C64) * c.astype(F32)
        S = (S + v).astype(C64)
    return S


def sp_coherence(S, defect=None):
    nchan = S.shape[0]
    Cg = np.ones((nchan, nchan, S.shape[2]), dtype=F32)
    for l in range(nchan):
        for m in range(nchan):
            if l == m:
                continue
            hi, lo = max(l, m), min(l, m)
            s = S[hi, lo] if defect != "coherence upper stride" else S.reshape(-1, S.shape[2], order="F")[(lo + hi * (nchan - 1)) % (nchan * nchan)]
            d1, d2 = S[hi, hi], S[lo, lo]
            Cg[l, m] = (np.abs(s) / np.sqrt((d1 * d2).real)).astype(F32)
    return Cg


def test_bound_passes_a_correct_single_precision_computation():
    rng = np.random.default_rng(1)
    worst = {}

    def note(k, r):
        worst[k] = max(worst.get(k, 0.0), r)

    for dt in (F32, C64):
        for su, sv, nf in (((300,), (41,), (340,)), ((20, 13), (5, 9), (24, 21)), ((6, 5, 4), (3, 2, 3), (8, 6, 6)),
                           ((900,), (132,), (1031,))):
            u, v = conv_data(rng, su, dt), conv_data(rng, sv, dt)
            note("conv_fft", check_elems(sp_conv_fft(u, v, nf, dt), hi_conv(u, v, dt), conv_bound(u, v, nf, dt)))
        for su, sv, nf in OS_SHAPES[:1] + OS_SHAPES[2:]:
            u, v = conv_data(rng, su, dt), conv_data(rng, sv, dt)
            note("conv_os", check_elems(sp_conv_os(u, v, nf, dt), hi_conv(u, v, dt), conv_bound(u, v, nf, dt)))
    for n in (1, 2, 3, 4, 5, 17, 1000, 1031, 4096):
        x = rng.standard_normal((n, 3)).astype(F32)
        y, ref, b = sp_hilbert(x), hilbert_ref(x, F32), hilbert_bound(x, F32)
        note("hilbert", check_elems(y, ref, b))
        note("hilbert", check_elems(y.real, x, b))
    for n1, n2, f1, f2 in PER2_SHAPES:
        s = per2_signal(rng, n1, n2, F32)
        r = float(n1 * n2)
        S, E = per2_ref(s, f1, f2, F32)
        note("per2_full", check_elems(sp_per2_full(s, f1, f2, r), S / r, power_bound(S, E, eps(F32), f1 * f2, 2) / r))
        tot, bnd, pop, _ = radial_ref(S, E, f1, f2, r, F32)
        note("per2_radial", check_radial(sp_per2_radial(s, f1, f2, r, False), sp_per2_radial(s, f1, f2, r, True),
                                         tot, bnd, pop, F32))
    for nchan, n, nfft, nt, weighted, demean in ((3, 256, 256, 3, False, True), (7, 1000, 1031, 7, True, False),
                                                 (2, 1024, 1024, 1, False, True)):
        rows = mt_tapers(n, nt, weighted)
        x = mt_signal(rng, nchan, n, F32, 1e3 if demean else 0.0)
        X, cf, dA = mt_ref(x, rows, nfft, demean, F32)
        nout = nfft // 2 + 1
        S, B = mt_cross_ref(X, cf, dA, 0, nout, F32)
        Sg = sp_mt_cross(x, rows, nfft, demean, 0, nout)
        note("mt_cross", check_elems(Sg, S, B))
        ref, lo, hi = coherence_interval(S, B, F32)
        note("mt_coherence", check_coherence(sp_coherence(Sg), ref, lo, hi))
    for k, r in sorted(worst.items()):
        print(f"largest error-to-bound ratio of a single-precision {k}: {r:.3g}")
    assert all(r < 1 for r in worst.values()) and len(worst) == 7


def _rejects(fn):
    try:
        fn()
    except AssertionError:
        return True
    return False


def test_bound_rejects_planted_defects():
    rng = np.random.default_rng(2)
    rejected = []

    def expect(name, fn):
        assert _rejects(fn), f"{name} passed the bound"
        rejected.append(name)

    # hilbert
    for n, defects in ((1000, ("nyquist doubled", "upper not zeroed", "no 1/n")), (1031, ("odd last not doubled",))):
        x = rng.standard_normal((n, 3)).astype(F32)
        ref, b = hilbert_ref(x, F32), hilbert_bound(x, F32)
        for d in defects:
            expect(f"hilbert: {d}", lambda: check_elems(sp_hilbert(x, d), ref, b))
    # 2-D periodogram
    s = per2_signal(rng, 40, 50, F32)
    S, E = per2_ref(s, 40, 50, F32)
    tot, bnd, pop, _ = radial_ref(S, E, 40, 50, 2000.0, F32)
    for d, name in (("nyquist row m2", "Nyquist row weighted m2"), ("c1 c2 swapped", "c1 and c2 swapped")):
        expect(f"per2: {name}", lambda: check_radial(sp_per2_radial(s, 40, 50, 2000.0, False, d),
                                                      sp_per2_radial(s, 40, 50, 2000.0, True, d), tot, bnd, pop, F32))
    s = per2_signal(rng, 37, 50, F32)
    S, E = per2_ref(s, 37, 50, F32)
    expect("per2: mirror index off by one (odd n1)",
           lambda: check_elems(sp_per2_full(s, 37, 50, 1850.0, "mirror off by one"), S / 1850.0,
                               power_bound(S, E, eps(F32), 37 * 50, 2) / 1850.0))
    # multitaper
    for nchan, n, nfft, f_lo, nf, defects in (
            (3, 256, 256, 0, 129, ("dc weight 2", "conj on a", "coherence upper stride")),
            (3, 1000, 1031, 0, 516, ("odd last weight 1",)),
            (3, 256, 256, 20, 60, ("f_lo ignored",))):
        rows = mt_tapers(n, 3, False)
        x = mt_signal(rng, nchan, n, F32, 0.0)
        X, cf, dA = mt_ref(x, rows, nfft, False, F32)
        S, B = mt_cross_ref(X, cf, dA, f_lo, nf, F32)
        ref, lo, hi = coherence_interval(S, B, F32)
        for d in defects:
            if d.startswith("coherence"):
                Sg = sp_mt_cross(x, rows, nfft, False, f_lo, nf)
                expect(f"mt: {d}", lambda: check_coherence(sp_coherence(Sg, d), ref, lo, hi))
            else:
                expect(f"mt: {d}", lambda: check_elems(sp_mt_cross(x, rows, nfft, False, f_lo, nf, d), S, B))
    # a demeaned bound does not pass an undemeaned signal
    rows = mt_tapers(256, 3, False)
    x = mt_signal(rng, 2, 256, F32, 1e3)
    X, cf, dA = mt_ref(x, rows, 256, True, F32)
    S, B = mt_cross_ref(X, cf, dA, 0, 129, F32)
    expect("mt: demean skipped", lambda: check_elems(sp_mt_cross(x, rows, 256, False, 0, 129), S, B))
    # N-D conv (overlap-save)
    for su, sv, nf in (((1000,), (37,), (128,)), ((40, 30), (7, 45), (16, 64)), ((12, 9, 10), (3, 4, 2), (8, 8, 4))):
        u, v = conv_data(rng, su, C64), conv_data(rng, sv, C64)
        ref, b = hi_conv(u, v, C64), conv_bound(u, v, nf, C64)
        expect(f"conv os {len(su)}-D: one block shifted by one sample",
               lambda: check_elems(sp_conv_os(u, v, nf, C64, shift_block=1), ref, b))
        expect(f"conv os {len(su)}-D: halo sv instead of sv - 1",
               lambda: check_elems(sp_conv_os(u, v, nf, C64, halo=lambda s: s), ref, b))
    for name in rejected:
        print("rejected:", name)
    assert rejected == [
        "hilbert: nyquist doubled", "hilbert: upper not zeroed", "hilbert: no 1/n", "hilbert: odd last not doubled",
        "per2: Nyquist row weighted m2", "per2: c1 and c2 swapped", "per2: mirror index off by one (odd n1)",
        "mt: dc weight 2", "mt: conj on a", "mt: coherence upper stride", "mt: odd last weight 1", "mt: f_lo ignored",
        "mt: demean skipped",
        "conv os 1-D: one block shifted by one sample", "conv os 1-D: halo sv instead of sv - 1",
        "conv os 2-D: one block shifted by one sample", "conv os 2-D: halo sv instead of sv - 1",
        "conv os 3-D: one block shifted by one sample", "conv os 3-D: halo sv instead of sv - 1"]


# =============================================================================== case tables

# (nu, nv, nfft) of conv_fft_exec: n = 1, 2, 3; nfft equal to the output size (odd and even); padded; non-smooth
CONV_FFT_CASES = [(1, 1, 1), (2, 1, 2), (2, 2, 3), (3, 2, 4), (500, 41, 540), (500, 40, 539), (300, 200, 512),
                  (900, 132, 1031), (1000, 1000, 1999)]
# (su, sv, nffts) of the N-D :fft_simple: rank 1-3, nffts equal to the output size, padded, non-smooth, v longer than u
ND_FFT_CASES = [((1,), (1,), (1,)), ((3,), (2,), (4,)), ((500,), (41,), (540,)), ((900,), (132,), (1031,)),
                ((33, 20), (5, 40), (37, 59)), ((33, 20), (5, 40), (40, 64)), ((1, 50), (1, 7), (1, 56)),
                ((9, 7, 5), (4, 3, 6), (12, 9, 10)), ((9, 7, 5), (4, 3, 6), (12, 10, 11))]
HILBERT_N = (1, 2, 3, 4, 5, 17, 1000, 1031, 4096, 65537)
HILBERT_COLS = (1, 3, 64)
# (n1, n2, nfft1, nfft2): square; n1 odd / even; f1 > f2, f1 < f2; zero padding; a prime nfft; 2x2, 2x3, 3x2; 2 x 4096
PER2_SHAPES = [(64, 64, 64, 64), (37, 50, 37, 50), (40, 50, 40, 50), (80, 45, 80, 45), (51, 40, 51, 40),
               (30, 20, 64, 48), (100, 30, 1031, 31), (2, 2, 2, 2), (2, 3, 2, 3), (3, 2, 3, 2), (2, 4096, 2, 4096)]
MT_FRANGES = ("none", "dc", "nyquist", "interior", "empty")


def mt_fused(dt, nfft):
    return 256 <= nfft <= (8192 if _f64(dt) else 16384) and nfft & (nfft - 1) == 0


def mt_cases(dt):
    """(nchan, n, nfft, ntapers, weighted, demean, frange) of test_mt_cross_spectra: fused powers of two and cuFFT sizes
    (odd and even), every channel count, taper count, weighting, demean and frequency range."""
    sizes = ((256, 256), (1024, 1000), (4096, 4096), (16384, 16384)) if not _f64(dt) else ((256, 256), (2048, 2000), (8192, 8192))
    sizes += ((1000, 1000), (1031, 1031), (1031, 999), (32768, 32768))
    cases = []
    for i, (nfft, n) in enumerate(sizes):
        nchan = (1, 2, 3, 7)[i % 4]
        nt = (1, 3, 7)[i % 3]
        cases.append((nchan, n, nfft, nt, i % 2 == 1, (i // 2) % 2 == 1, MT_FRANGES[i % 5]))
    cases.append((3, 512, 512, 3, True, True, "nyquist"))
    cases.append((7, 300, 300, 3, False, True, "empty"))
    cases.append((2, 256, 256, 7, True, False, "interior"))
    return cases


def mt_range(frange, nout):
    return {"none": (0, nout), "dc": (0, nout // 3), "nyquist": (nout // 2, nout - nout // 2),
            "interior": (nout // 4, nout // 3), "empty": (nout // 2, 0)}[frange]


def test_case_table_covers_every_instance():
    # convolutions: every eltype runs every case; the cases reach n = 1, 2, 3, nfft == output (odd and even), non-smooth
    reach = set()
    for nu, nv, nfft in CONV_FFT_CASES:
        reach |= {("fft", "exact" if nfft == nu + nv - 1 else "padded"), ("fft", "odd" if nfft % 2 else "even"),
                  ("fft", "nonsmooth" if nonsmooth([nfft]) else "smooth")}
    assert {nu for nu, _, _ in CONV_FFT_CASES} >= {1, 2, 3}
    for su, sv, nf in ND_FFT_CASES:
        so = [a + b - 1 for a, b in zip(su, sv)]
        reach |= {("nd", len(su)), ("nd", "exact" if list(nf) == so else "padded"), ("nd", "odd" if nf[0] % 2 else "even"),
                  ("nd", "nonsmooth" if nonsmooth(nf) else "smooth")}
        assert all(f >= o for f, o in zip(nf, so))
    assert any(any(b > a for a, b in zip(su, sv)) for su, sv, _ in ND_FFT_CASES)
    for dt in DTYPES:
        for su, sv, nf, regime in os_cases(dt):
            reach |= {("os", dt.name, regime), ("os", len(su))}
    want = {(k, v) for k in ("fft", "nd") for v in ("exact", "padded", "odd", "even", "nonsmooth", "smooth")}
    want |= {("nd", r) for r in (1, 2, 3)} | {("os", r) for r in (1, 2, 3)}
    want |= {("os", dt.name, r) for dt in DTYPES for r in OS_REGIMES}
    assert want <= reach, sorted(want - reach, key=str)
    # hilbert: n = 1, 2, 3, odd and even, non-smooth, several columns
    assert {n % 2 for n in HILBERT_N} == {0, 1} and {1, 2, 3} <= set(HILBERT_N) and any(nonsmooth([n]) for n in HILBERT_N)
    # periodogram: odd / even n1, f1 > f2 / f1 < f2 / square, padding, prime nfft, the tiny shapes and a tall one
    kinds = set()
    for n1, n2, f1, f2 in PER2_SHAPES:
        kinds |= {"odd n1" if f1 % 2 else "even n1", "f1>f2" if f1 > f2 else "f1<f2" if f1 < f2 else "square"}
        kinds |= {"padded"} if (n1, n2) != (f1, f2) else set()
        kinds |= {"prime"} if nonsmooth([f1, f2]) else set()
    assert kinds == {"odd n1", "even n1", "f1>f2", "f1<f2", "square", "padded", "prime"}
    assert {(2, 2), (2, 3), (3, 2), (2, 4096)} <= {(a, b) for a, b, _, _ in PER2_SHAPES}
    # multitaper: (eltype, route, nfft parity) and every option value
    combos, opts = set(), set()
    for dt in REALS:
        for nchan, n, nfft, nt, w, dm, fr in mt_cases(dt):
            combos.add((dt.name, "fused" if mt_fused(dt, nfft) else "cufft", nfft % 2, n % 2))
            opts |= {("nchan", nchan), ("nt", nt), ("w", w), ("demean", dm), ("fr", fr)}
            opts |= {("fused nfft", dt.name, nfft)} if mt_fused(dt, nfft) else {("cufft nfft", nfft)}
    for dt in REALS:
        assert {(dt.name, "fused", 0, 0), (dt.name, "cufft", 0, 0), (dt.name, "cufft", 1, 1)} <= combos, combos
    assert {("nchan", c) for c in (1, 2, 3, 7)} | {("nt", t) for t in (1, 3, 7)} | {("w", True), ("w", False)} | \
        {("demean", True), ("demean", False)} | {("fr", f) for f in MT_FRANGES} <= opts
    assert {("fused nfft", "float32", 256), ("fused nfft", "float32", 16384), ("fused nfft", "float64", 8192)} <= opts
    assert {("cufft nfft", n) for n in (1000, 1031, 32768)} <= opts
    for f in MT_FRANGES:
        lo, nf = mt_range(f, 129)
        assert 0 <= lo and lo + nf <= 129
    assert mt_range("dc", 129)[0] == 0 and sum(mt_range("nyquist", 129)) == 129 and mt_range("empty", 129)[1] == 0


# =============================================================================== GPU helpers

@pytest.fixture(scope="module")
def dsp():
    return pytest.importorskip("dspb200")


class Guarded:
    """A device buffer of GUARD cells, `n` data cells and GUARD cells: sentinels of magnitude 10^6 (input, rng given) or
    NaN (output) outside the data."""

    def __init__(self, dt, n, rng=None, data=None):
        from dspb200 import device
        self.dt, self.n, self.lo = np.dtype(dt), n, GUARD
        total = n + 2 * GUARD
        if rng is None:
            host = np.full(total, np.nan, dtype=dt)
        else:
            s = rng.choice(np.array([-SENTINEL, SENTINEL]), total)
            if _cplx(dt):
                s = s + 1j * rng.choice(np.array([-SENTINEL, SENTINEL]), total)
            host = s.astype(dt)
        if data is not None:
            host[GUARD:GUARD + n] = np.asarray(data).ravel(order="F")
        self.host = host
        self.buf = device.to_device(host)
        self.ptr = self.buf.ptr + GUARD * self.dt.itemsize

    def data(self, shape=None):
        """The data cells (Fortran-ordered `shape`), after checking that the cells around them are unchanged."""
        h = self.buf.to_host()
        outside = np.concatenate([h[:GUARD], h[GUARD + self.n:]])
        want = np.concatenate([self.host[:GUARD], self.host[GUARD + self.n:]])
        assert np.array_equal(outside, want, equal_nan=True), "a cell outside the buffer's range changed"
        d = h[GUARD:GUARD + self.n]
        return d if shape is None else d.reshape(shape, order="F")


class HostOut:
    """A host output of n cells followed by GUARD NaN cells that must survive the call."""

    def __init__(self, dt, n):
        self.n = n
        self.buf = np.full(n + GUARD, np.nan, dtype=dt)
        self.ptr = self.buf.ctypes.data_as(C.c_void_p)

    def data(self, shape=None):
        assert np.isnan(self.buf[self.n:]).all(), "a host cell past the output changed"
        d = self.buf[:self.n]
        return d if shape is None else d.reshape(shape, order="F")


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype.itemsize in (8, 16) else np.uint32)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _code(dsp, dt):
    return dsp._lib.np_dtype_code(np.dtype(dt))


def _i64(vals):
    return np.asarray(vals, dtype=np.int64)


_RATIOS = {}


def _note(family, dt, ratio, sizes=()):
    key = (family, _real(dt).name, "non-smooth" if nonsmooth(sizes) else "")
    _RATIOS[key] = max(_RATIOS.get(key, 0.0), ratio)


# =============================================================================== GPU: convolutions

def _conv_nd_dev(dsp, dt, u, v, nf, overlapsave, rng):
    from dspb200 import device
    so = tuple(a + b - 1 for a, b in zip(u.shape, v.shape))
    gu, gv = Guarded(dt, u.size, rng, u), Guarded(dt, v.size, rng, v)
    go = Guarded(dt, int(np.prod(so)))
    us, vs, nfs = _i64(u.shape), _i64(v.shape), _i64(nf)
    fn = dsp._lib.lib.dspb200_conv_nd_os_exec_dev if overlapsave else dsp._lib.lib.dspb200_conv_nd_exec_dev
    dsp._lib.check(fn(_code(dsp, dt), u.ndim, dsp._lib.ptr(us), gu.ptr, dsp._lib.ptr(vs), gv.ptr, dsp._lib.ptr(nfs), go.ptr,
                      None))
    device.sync()
    gu.data()
    gv.data()
    return go.data(so)


def _conv_nd_host(dsp, dt, u, v, nf, overlapsave):
    so = tuple(a + b - 1 for a, b in zip(u.shape, v.shape))
    uf, vf = np.asfortranarray(u), np.asfortranarray(v)
    us, vs, nfs = _i64(u.shape), _i64(v.shape), _i64(nf)
    out = HostOut(dt, int(np.prod(so)))
    fn = dsp._lib.lib.dspb200_conv_nd_os_exec if overlapsave else dsp._lib.lib.dspb200_conv_nd_exec
    dsp._lib.check(fn(_code(dsp, dt), u.ndim, dsp._lib.ptr(us), dsp._lib.ptr(uf), dsp._lib.ptr(vs), dsp._lib.ptr(vf),
                      dsp._lib.ptr(nfs), out.ptr))
    return out.data(so)


def _check_conv(y, u, v, nf, dt, integer, what):
    if integer:
        ex = int_conv(u, v)
        assert np.array_equal(np.rint(y.real), ex.real), what
        assert not _cplx(dt) or np.array_equal(np.rint(y.imag), ex.imag), what
        ref = ex
    else:
        ref = hi_conv(u, v, dt)
    return check_elems(y, ref, conv_bound(u, v, nf, dt), what)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_conv_fft_exec(dsp, dt):
    """The 1-D :fft_simple of the Julia glue: exact on integers, bounded on random data, and bit-identical to the rank-1
    N-D :fft_simple on device pointers (the same cached cuFFT plan, the same scaling and product kernels)."""
    from dspb200 import device
    rng = np.random.default_rng([dt.num, 1])
    try:
        for nu, nv, nfft in CONV_FFT_CASES:
            for integer in (True, False):
                u, v = conv_pair(rng, (nu,), (nv,), (nfft,), dt, integer)
                out = HostOut(dt, nu + nv - 1)
                dsp._lib.check(dsp._lib.lib.dspb200_conv_fft_exec(_code(dsp, dt), dsp._lib.ptr(u), nu, dsp._lib.ptr(v), nv,
                                                                  nfft, out.ptr))
                y = out.data()
                _note("conv_fft", dt, _check_conv(y, u, v, (nfft,), dt, integer, (nu, nv, nfft, integer)), (nfft,))
                yd = _conv_nd_dev(dsp, dt, u, v, (nfft,), False, rng)
                assert same_bits(y, yd), (nu, nv, nfft, integer)
    finally:
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_conv_nd_fft(dsp, dt):
    from dspb200 import device
    rng = np.random.default_rng([dt.num, 2])
    try:
        for su, sv, nf in ND_FFT_CASES:
            for integer in (True, False):
                u, v = conv_pair(rng, su, sv, nf, dt, integer)
                y = _conv_nd_host(dsp, dt, u, v, nf, False)
                _note("conv_nd", dt, _check_conv(y, u, v, nf, dt, integer, (su, sv, nf, integer)), nf)
                assert same_bits(y, _conv_nd_dev(dsp, dt, u, v, nf, False, rng)), (su, sv, nf, integer)
    finally:
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_conv_nd_os(dsp, dt):
    from dspb200 import device
    rng = np.random.default_rng([dt.num, 3])
    try:
        for su, sv, nf, regime in os_cases(dt):
            dsp._lib.conv_nd_os_set_budget(os_budget(dt, su, sv, nf, regime))
            for integer in (True, False):
                u, v = conv_pair(rng, su, sv, nf, dt, integer)
                y = _conv_nd_host(dsp, dt, u, v, nf, True)
                _note("conv_nd_os", dt, _check_conv(y, u, v, nf, dt, integer, (su, sv, nf, regime, integer)), nf)
                assert same_bits(y, _conv_nd_dev(dsp, dt, u, v, nf, True, rng)), (su, sv, nf, regime, integer)
    finally:
        dsp._lib.conv_nd_os_set_budget(DEFAULT_BUDGET)
        device.empty_cache()


# =============================================================================== GPU: hilbert

@pytest.mark.gpu
@pytest.mark.parametrize("dt", REALS, ids=lambda d: d.name)
def test_hilbert(dsp, dt):
    from dspb200 import device
    rng = np.random.default_rng([dt.num, 4])
    try:
        for n in HILBERT_N:
            for ncols in HILBERT_COLS:
                x = (rng.standard_normal((n, ncols)) * rng.uniform(0.01, 100, ncols)[None, :]).astype(dt)
                gx = Guarded(dt, x.size, rng, x)
                go = Guarded(_ccx(dt), x.size)
                dsp._lib.check(dsp._lib.lib.dspb200_hilbert_exec_dev(_code(dsp, dt), gx.ptr, n, ncols, go.ptr, None))
                device.sync()
                gx.data()
                yd = go.data((n, ncols))
                out = HostOut(_ccx(dt), x.size)
                xf = np.asfortranarray(x)
                dsp._lib.check(dsp._lib.lib.dspb200_hilbert_exec(_code(dsp, dt), dsp._lib.ptr(xf), n, ncols, out.ptr))
                y = out.data((n, ncols))
                assert same_bits(y, yd), (n, ncols)
                b = hilbert_bound(x, dt)
                _note("hilbert", dt, check_elems(y, hilbert_ref(x, dt), b, (n, ncols)), (n,))
                _note("hilbert", dt, check_elems(y.real, x, b, ("Re", n, ncols)), (n,))
    finally:
        device.empty_cache()


# =============================================================================== GPU: 2-D periodogram

@pytest.mark.gpu
@pytest.mark.parametrize("dt", REALS, ids=lambda d: d.name)
def test_periodogram2(dsp, dt):
    from dspb200 import device
    rng = np.random.default_rng([dt.num, 5])
    try:
        for n1, n2, f1, f2 in PER2_SHAPES:
            s = per2_signal(rng, n1, n2, dt)
            r = float(n1 * n2) * 2.5                               # fs = 2.5
            S, E = per2_ref(s, f1, f2, dt)
            tot, bnd, pop, kmax = radial_ref(S, E, f1, f2, r, dt)
            assert (pop > 0).all()
            gs = Guarded(dt, s.size, rng, s)
            sf = np.asfortranarray(s)
            res = {}
            for ptype in (0, 1, 2):
                nout = f1 * f2 if ptype == 0 else kmax
                go = Guarded(_real(dt), nout)
                dsp._lib.check(dsp._lib.lib.dspb200_periodogram2_exec_dev(_code(dsp, dt), gs.ptr, n1, n2, f1, f2, r, ptype,
                                                                          go.ptr, None))
                device.sync()
                gs.data()
                out = HostOut(_real(dt), nout)
                dsp._lib.check(dsp._lib.lib.dspb200_periodogram2_exec(_code(dsp, dt), dsp._lib.ptr(sf), n1, n2, f1, f2, r,
                                                                      ptype, out.ptr))
                res[ptype] = (out.data(), go.data())
            (Ph, Pd) = res[0]
            assert same_bits(Ph, Pd), (n1, n2, f1, f2)
            pb = power_bound(S, E, eps(dt), f1 * f2, 2) / r
            _note("per2_full", dt, check_elems(Ph.reshape((f1, f2), order="F"), S / r, pb, (n1, n2, f1, f2)), (f1, f2))
            for k in (0, 1):                                       # host, device: not bitwise (Float64 atomics)
                _note("per2_radial", dt, check_radial(res[1][k], res[2][k], tot, bnd, pop, dt, (n1, n2, f1, f2, k)), (f1, f2))
    finally:
        device.empty_cache()


# =============================================================================== GPU: multitaper cross spectra

@pytest.mark.gpu
@pytest.mark.parametrize("dt", REALS, ids=lambda d: d.name)
def test_mt_cross_spectra(dsp, dt):
    from dspb200 import device
    rng = np.random.default_rng([dt.num, 7])
    try:
        for case in mt_cases(dt):
            nchan, n, nfft, nt, weighted, demean, frange = case
            rows = mt_tapers(n, nt, weighted)
            x = mt_signal(rng, nchan, n, dt, 1e3 if demean else 0.0)
            nout = nfft // 2 + 1
            f_lo, nf = mt_range(frange, nout)
            mt = dsp._lib.MtPlan(dt, n, 0, nfft, True, rows)
            try:
                assert mt.fused == mt_fused(dt, nfft) and mt.nout == nout
                gx = Guarded(dt, x.size, rng, x)                   # the n_channels x n_samples matrix, channel fastest
                xf = np.asfortranarray(x)
                got = {}
                for coh in (False, True):
                    odt = _real(dt) if coh else _ccx(dt)
                    cnt = nchan * nchan * nf
                    go = Guarded(odt, cnt)
                    dsp._lib.check(dsp._lib.lib.dspb200_mt_cross_spectra_exec_dev(mt.handle, gx.ptr, nchan, int(demean), f_lo,
                                                                                  nf, int(coh), go.ptr, None))
                    device.sync()
                    gx.data()
                    out = HostOut(odt, cnt)
                    dsp._lib.check(dsp._lib.lib.dspb200_mt_cross_spectra_exec(mt.handle, dsp._lib.ptr(xf), nchan,
                                                                              int(demean), f_lo, nf, int(coh), out.ptr))
                    h, d = out.data((nchan, nchan, nf)), go.data((nchan, nchan, nf))
                    if nf == 0:                                    # nothing written: the NaN cells survive
                        assert h.size == 0 and d.size == 0
                    assert same_bits(h, d), (case, coh)
                    got[coh] = h
                if nf == 0:
                    continue
                X, cf, dA = mt_ref(x, rows, nfft, demean, dt)
                S, B = mt_cross_ref(X, cf, dA, f_lo, nf, dt)
                _note("mt_cross", dt, check_elems(got[False], S, B, case), (nfft,))
                for l in range(nchan):                             # the diagonal's imaginary part, under the same bound
                    assert (np.abs(got[False][l, l].imag) <= B[l, l]).all(), case
                ref, lo, hi = coherence_interval(S, B, dt)
                Cg = got[True]
                _note("mt_coherence", dt, check_coherence(Cg.astype(np.float64), ref, lo, hi, case), (nfft,))
                assert same_bits(Cg, Cg.transpose(1, 0, 2)), case              # both read one lower-triangle entry
            finally:
                mt.close()
    finally:
        device.empty_cache()


@pytest.mark.gpu
def test_report_largest_ratio():
    # runs last in this module: the largest error-to-bound ratio seen per family, eltype and size class
    for (family, dt, cls), ratio in sorted(_RATIOS.items()):
        print(f"largest error-to-bound ratio {family:13s} {dt:8s} {cls:10s}: {ratio:.3g}")
    assert _RATIOS and all(r <= 1.0 for r in _RATIOS.values())
