"""Every time-domain FIR and direct-convolution kernel instance and entry point, bit for bit against the reference's
fused multiply-add chain.

Both kernel families promise the reference's arithmetic one `muladd` at a time, which on FMA hardware is one correctly
rounded fused multiply-add per step (Base.muladd for Complex: two fmas per part, base/complex.jl):
* `fir_tile_kernel<E, NT, STATE>` (fir.cu, fir_tile.cuh), 16 instances: 4 eltypes x 128 / 256 threads x STATE.  Output i is
  the chain over the taps oldest first, y = fma(x[i], b[0], fma(x[i-1], b[1], ... fma(x[i-nb+1], b[nb-1], seed))), the
  seed being the incoming state for i < nb - 1 (STATE) and zero otherwise; samples outside the call are zero.  For real
  eltypes that is the reference's _filt_fir! (src/dspbase.jl:95-141).  For complex ones the reference forms the last tap's
  term b[nb] * x as a plain complex product where the kernel fuses it (DESIGN section 4): the kernel is checked against
  its own documented chain, and the difference is pinned on the CPU.
* `conv_direct_nd_kernel` (overlap_save.cu), ranks 1-3, 1-D also through `dspb200_conv_direct_exec`: _conv_td!
  (src/dspbase.jl:646-660).  Its loop `for m in CartesianIndices(u), n in CartesianIndices(v)` (n outer instead when
  size(u,1) > size(v,1)) has the FIRST iterator outside, so each output sums its products in the column-major order of the
  outer array's index, each step muladd(u[m], v[n], acc).

The restated chains below are vectorised over outputs, one numpy step per tap (or per outer index), with exact fmas
(oracle.dspbase.fma_f32 / fma_f64 / cmuladd), which are themselves pinned against fractions.Fraction; on small shapes
the restatements are pinned against literal nested-loop transcriptions of the Julia source in Fraction arithmetic.
Planted defects (reversed order, an unfused multiply-add, a chain shifted by one tap, swapped complex operands, a
skipped padding-chunk tap) must each change an output bit on the test data: samples and taps are normals scaled by 2^k,
k uniform in [-20, 20], so roundings depend on the order.  The routing (fir_launch's 128 / 256-thread rule) and the
per-instance geometry (fir_geom) are restated so that the CPU can show what the case table reaches.

GPU checks are array_equal: device calls run between NaN output cells with +-1000 sentinel samples around the input."""
import zlib
from fractions import Fraction

import numpy as np
import pytest

from oracle import dspbase as od

F32, F64, C64, C128 = (np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))
DTYPES = (F32, F64, C64, C128)
CPU_SMS = 132             # the H100's SM count: the routing the CPU restates
KC = 512                  # taps per staging round (fir_geom::KC)
GUARD = 64                # sentinel / NaN cells on each side of a device buffer
SPREAD = 20               # data: normal * 2^k, k uniform in [-SPREAD, SPREAD]


def _cplx(dt):
    return np.dtype(dt).kind == "c"


def _real(dt):
    return {F32: F32, F64: F64, C64: F32, C128: F64}[np.dtype(dt)]


def _cdiv(a, b):
    return -(-a // b)


# =============================================================================== exact arithmetic (fractions.Fraction)

def _q(a):
    return Fraction(float(a))


def _round_q(q, R):
    """The real dtype R's nearest value to the rational q, ties to even.  Valid domain: q zero or a normal number of R."""
    R = np.dtype(R)
    tiny, big = np.finfo(R).tiny, np.finfo(R).max
    assert q == 0 or float(tiny) <= abs(q) <= float(big), "outside the valid domain: subnormal or overflowing result"
    r = float(q)                                            # correctly rounded to Float64 (integer true division)
    if R == F64:
        return np.float64(r)
    c = np.float32(r)
    if float(c) == r:                                       # the Float64 rounding is a Float32: q is within half a Float64 ulp
        return c
    best = None
    for cand in (np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf))):
        d = abs(_q(cand) - q)
        if best is None or d < best[0] or (d == best[0] and int(cand.view(np.int32)) & 1 == 0):
            best = (d, cand)
    return best[1]


def _fma_q(a, b, c, R):
    return _round_q(_q(a) * _q(b) + _q(c), R)


def _muladd_q(a, b, c, T):
    """muladd(a, b, c) in eltype T, every fma rounded once from the exact value; complex: Base.muladd."""
    T = np.dtype(T)
    if not _cplx(T):
        return _fma_q(a, b, c, T)
    R = _real(T)
    re = _fma_q(a.real, b.real, -_fma_q(a.imag, b.imag, -c.real, R), R)
    im = _fma_q(a.real, b.imag, _fma_q(a.imag, b.real, c.imag, R), R)
    return T.type(complex(re, im))


def _mul_q(a, b, T):
    """a * b in eltype T without fusion (Julia's Complex * : each product rounded, then the sum)."""
    T = np.dtype(T)
    if not _cplx(T):
        return _round_q(_q(a) * _q(b), T)
    R = _real(T)
    re = _round_q(_q(_round_q(_q(a.real) * _q(b.real), R)) - _q(_round_q(_q(a.imag) * _q(b.imag), R)), R)
    im = _round_q(_q(_round_q(_q(a.real) * _q(b.imag), R)) + _q(_round_q(_q(a.imag) * _q(b.real), R)), R)
    return T.type(complex(re, im))


# =============================================================================== test data

def _data(rng, shape, dt, spread=SPREAD):
    """Normals scaled by 2^k, k uniform in [-spread, spread] (both parts of complex data, independently)."""
    def part():
        return rng.standard_normal(shape) * np.exp2(rng.integers(-spread, spread + 1, shape))
    v = part() + 1j * part() if _cplx(dt) else part()
    return np.asarray(v).astype(dt)


def _triples(rng, n, R, E):
    """n (a, b, c) triples of the real dtype R: exponent spread +-E, cancellations c = -(a*b rounded) (+ a small term),
    exact ties (a*b exact in R, c half an ulp of it) and near ties (that half ulp +- a tiny amount), zeros."""
    R = np.dtype(R)
    p = np.finfo(R).nmant + 1

    def rnd(m):
        return (rng.choice([-1.0, 1.0], m) * rng.uniform(1, 2, m) * np.exp2(rng.integers(-E, E + 1, m))).astype(R)
    a, b, c = rnd(n), rnd(n), rnd(n)
    q = n // 5
    sl = slice(0, q)                                        # cancellations
    prod = (a[sl].astype(np.float64) * b[sl].astype(np.float64)).astype(R)
    c[sl] = -prod
    c[q // 2: q] = (-prod[q // 2:].astype(np.float64) * (1 + np.exp2(-p + 2) * rng.integers(-4, 5, q - q // 2))).astype(R)
    sl = slice(q, 3 * q)                                    # ties and near ties: a, b with p // 2 - 1 significant bits
    h = p // 2 - 1
    ma = rng.integers(2 ** (h - 1), 2 ** h, 2 * q)
    mb = rng.integers(2 ** (h - 1), 2 ** h, 2 * q)
    ea, eb = rng.integers(-E // 2, E // 2 + 1, 2 * q), rng.integers(-E // 2, E // 2 + 1, 2 * q)
    a[sl] = (rng.choice([-1.0, 1.0], 2 * q) * ma * np.exp2(ea - h)).astype(R)
    b[sl] = (mb * np.exp2(eb - h)).astype(R)
    pr = a[sl].astype(np.float64) * b[sl].astype(np.float64)        # exact in R
    half_ulp = np.exp2(np.floor(np.log2(np.abs(pr))) - p)
    sgn = rng.choice([-1.0, 1.0], 2 * q)
    nudge = np.where(np.arange(2 * q) % 2 == 0, 0.0, rng.choice([-1.0, 1.0], 2 * q) * np.exp2(-p // 2))
    c[sl] = (sgn * half_ulp * (1 + nudge)).astype(R)
    z = slice(3 * q, 3 * q + 50)                            # zeros in every position
    a[z][::3], b[z][1::3], c[z][2::3] = 0, 0, 0
    return a, b, c


# =============================================================================== restated chains

def _plain_mul(x, b, E):
    """x * b in eltype E without fusion (separate numpy operations: one rounding each)."""
    if not _cplx(E):
        return np.multiply(x, b, dtype=E)
    R = _real(E)
    x, b = np.broadcast_arrays(np.asarray(x, dtype=E), np.asarray(b, dtype=E))
    xr, xi, br, bi = x.real, x.imag, b.real, b.imag
    out = np.empty(x.shape, dtype=E)
    out.real = np.subtract(np.multiply(xr, br), np.multiply(xi, bi))
    out.imag = np.add(np.multiply(xr, bi), np.multiply(xi, br))
    return out


def fir_chain(b, x, si=None, state=False, plain_last=False, defect=None):
    """The FIR chains of one call, vectorised over the outputs (one numpy step per tap).

    x: (nx, ncols) in eltype E, b: (nb,), si: (nb - 1, ncols) or None (zero).  Outputs i in [0, nout), nout = nx, or
    nx + nb - 1 with `state` (the last nb - 1 are the final state).  The kernel's chain: acc = si[i] for i < nb - 1 (else
    0), then acc = muladd(x[i - k], b[k], acc) for k = nb - 1 .. 0, x zero outside [0, nx).  plain_last: the reference's
    chain, whose tap nb - 1 term is the plain product b[nb] * x when its sample lies in the call (i >= nb - 1); the same
    as the kernel's for real eltypes.  defect: 'reversed', 'unfused', 'shift' (each tap one sample late), 'swap'
    (muladd(b, x, acc)) or 'skip_pad' (the oldest tap, the first real tap of the padding chunk when nb % 8, left out).
    Returns (y, si_out) (si_out None without `state`)."""
    E = x.dtype
    nb = b.size
    ns = nb - 1
    nx, ncols = x.shape
    nout = nx + ns if state else nx
    acc = np.zeros((nout, ncols), dtype=E)
    if si is not None:
        acc[:ns] = si
    xp = np.concatenate([np.zeros((ns + 1, ncols), E), x, np.zeros((ns + 1, ncols), E)])     # xp[ns + 1 + j] = x[j]
    taps = range(nb) if defect == "reversed" else range(ns, -1, -1)
    for k in taps:
        if defect == "skip_pad" and k == ns:
            continue
        off = ns + 1 - k + (1 if defect == "shift" else 0)
        seg = xp[off: off + nout]
        if defect == "unfused":
            acc = np.add(_plain_mul(seg, b[k], E), acc)
        elif defect == "swap":
            acc = od.cmuladd(np.broadcast_to(b[k], seg.shape), seg, acc)
        else:
            acc = od.muladd(seg, b[k], acc, E)
        if plain_last and k == ns and _cplx(E) and nout > ns:
            acc[ns:] = _plain_mul(seg[ns:], b[k], E)
    return (acc[:nx], acc[nx:]) if state else (acc, None)


def fir_literal(b, x, si, plain_last):
    """_filt_fir!, src/dspbase.jl:95-105, on one column, literally: the state carried in and out, every muladd one exact
    rounding (Fraction).  plain_last: si[silen] = b[silen + 1] * xi as the reference writes it; else muladd(xi, b, 0), the
    kernel's chain.  Returns (y, si_out)."""
    T = x.dtype
    si = np.array(si, dtype=T, copy=True)
    silen = b.size - 1
    zero = T.type(0)
    y = np.empty(x.size, dtype=T)
    last = (lambda xi, bb: _mul_q(bb, xi, T)) if plain_last else (lambda xi, bb: _muladd_q(xi, bb, zero, T))
    for i, xi in enumerate(x):
        if silen == 0:
            y[i] = last(xi, b[0])
            continue
        y[i] = _muladd_q(xi, b[0], si[0], T)
        for j in range(silen - 1):
            si[j] = _muladd_q(xi, b[j + 1], si[j + 1], T)
        si[silen - 1] = last(xi, b[silen])
    return y, si


def _cartesian(shape):
    """CartesianIndices(shape) in Julia's order: dim 1 fastest."""
    return [idx[::-1] for idx in np.ndindex(*shape[::-1])]


def conv_chain(u, v, walk, reverse=False, fused=True, swap=False):
    """Direct convolution of equal-rank arrays, vectorised: one step per index of the `walk` array ('u' or 'v') in
    column-major order (reversed with `reverse`), adding muladd(u[m], v[n], acc) (swap: muladd(v[n], u[m], acc); not
    fused: the product rounded, then the sum) to every output that index reaches."""
    T = np.result_type(u, v)
    u, v = u.astype(T), v.astype(T)
    out = np.zeros(tuple(a + b - 1 for a, b in zip(u.shape, v.shape)), dtype=T)
    outer, inner = (u, v) if walk == "u" else (v, u)
    idx = _cartesian(outer.shape)
    for m in (idx[::-1] if reverse else idx):
        sl = tuple(slice(i, i + n) for i, n in zip(m, inner.shape))
        a, bb = (outer[m], inner) if walk == "u" else (inner, outer[m])      # a from u, bb from v
        if not fused:
            out[sl] = np.add(_plain_mul(a, bb, T), out[sl])
        elif swap and _cplx(T):                             # (a real fma does not depend on its operands' order)
            out[sl] = od.cmuladd(*np.broadcast_arrays(bb, a), out[sl])
        else:
            out[sl] = od.muladd(a, bb, out[sl], T)
    return out


def conv_walk(u, v):
    """The reference's outer array: u when size(u,1) <= size(v,1) (src/dspbase.jl:650)."""
    return "u" if u.shape[0] <= v.shape[0] else "v"


def conv_literal(u, v):
    """_conv_td!, src/dspbase.jl:646-660, literally: the two nested Cartesian loops, first iterator outer, one exact
    rounding per muladd (Fraction)."""
    T = np.result_type(u, v)
    u, v = u.astype(T), v.astype(T)
    out = np.zeros(tuple(a + b - 1 for a, b in zip(u.shape, v.shape)), dtype=T)
    if u.shape[0] <= v.shape[0]:
        pairs = ((m, n) for m in _cartesian(u.shape) for n in _cartesian(v.shape))
    else:
        pairs = ((m, n) for n in _cartesian(v.shape) for m in _cartesian(u.shape))
    for m, n in pairs:
        k = tuple(a + b for a, b in zip(m, n))
        out[k] = _muladd_q(u[m], v[n], out[k], T)
    return out


# =============================================================================== routing and geometry restated from fir.cu

def fir_geom(dt, NT):
    """fir_geom<E, NT> (fir_tile.cuh:37-47): (G outputs per thread, TILE outputs per CTA)."""
    G = 4 if np.dtype(dt).itemsize == 16 else 8
    return G, NT * G


def fir_nt(dt, nout, ncols, sms=CPU_SMS):
    """fir_launch (fir.cu:76-86): 128-thread tiles when the 256-thread grid would not cover every SM eight times."""
    return 128 if _cdiv(nout, fir_geom(dt, 256)[1]) * ncols < 8 * sms else 256


def fir_rounds(nb):
    """kc of every staging round: taps padded at the old end to nb8 = a multiple of 8, KC = 512 per round."""
    nb8 = (nb + 7) & ~7
    kcs, k_hi = [], nb8 - 1
    while k_hi >= 0:
        kcs.append(min(k_hi + 1, KC))
        k_hi -= KC
    return kcs


def fir_instance(dt, nb, nx, ncols, state, sms=CPU_SMS):
    """(dtype, NT, STATE) of the launch; a stateful call with nb == 1 has no state and runs the stateless kernel."""
    st = state and nb > 1
    nout = nx + nb - 1 if st else nx
    return np.dtype(dt), fir_nt(dt, nout, ncols, sms), st


def fir_features(dt, nb, nx, ncols, offset=0):
    """What a launch reaches: the store paths (uint4 store; scalar tail, a thread with i < nx < i + G; a column that starts
    off a 16-byte boundary -- `offset` elements is column 0's), the padding chunk or none, the number of staging rounds
    and a kc = 8 (mod 16) tail chunk.  Every thread of a column shares the column's alignment (G elements are 32 or 64
    bytes)."""
    dt = np.dtype(dt)
    G, _ = fir_geom(dt, 128)
    nb8 = (nb + 7) & ~7
    pad = nb8 != nb
    kcs = fir_rounds(nb)
    f = {"pad_chunk" if pad else "no_pad_chunk", f"rounds{len(kcs)}"}
    if any((kc - (8 if r == 0 and pad else 0)) % 16 == 8 for r, kc in enumerate(kcs)):
        f.add("tail8")
    aligned = [((offset + c * nx) * dt.itemsize) % 16 == 0 for c in range(min(ncols, 16))]
    if any(aligned) and nx >= G:
        f.add("uint4")
    if nx % G:
        f.add("scalar_tail")
    if not all(aligned):
        f.add("unaligned_col")
    return f


def _needed(dt):
    need = {"uint4", "scalar_tail", "pad_chunk", "no_pad_chunk", "rounds1", "rounds2", "rounds3", "tail8"}
    if np.dtype(dt).itemsize < 16:                          # a ComplexF64 element is 16 bytes: every column is aligned
        need.add("unaligned_col")
    return need


def _nx_values(dt):
    G, T1 = fir_geom(dt, 128)
    return [1, G - 1, G, T1 - 1, T1 + 1, 2 * T1 + G + 1]


NB_128 = (1, 7, 9, 17, 66, 512, 520, 1031)                # the tap counts, split between the two thread counts
NB_256 = (2, 8, 16, 67, 511, 513, 521, 1025)


def fir_cases(sms=CPU_SMS):
    """(dt, nb, nx, ncols, state, offset) for every instance.  Tap counts from 511 on take nx <= TILE + 1 (the
    reference costs nb per output); the 256-thread cases take as many columns as the rule needs (their data repeats
    with period 7, so the reference is computed on 7 columns)."""
    cases = []
    for dt in DTYPES:
        G, T1 = fir_geom(dt, 128)
        nxs = _nx_values(dt)
        for state in (False, True):
            for NT, nbs in ((128, NB_128), (256, NB_256)):
                for j, nb in enumerate(nbs):
                    if state and nb == 1:
                        nb = 2
                    nx = nxs[j % len(nxs)] if nb < 511 else (G - 1, T1 - 1, T1 + 1)[j % 3]
                    if nb >= 511 and j % 4 == 3:
                        nx = nb // 2 + 1                    # nx < nb - 1: a state longer than the chunk
                    ncols = (1, 3, 70)[j % 3]
                    nout = nx + nb - 1 if state else nx
                    if NT == 256:
                        ncols = max(ncols, _cdiv(8 * sms, _cdiv(nout, fir_geom(dt, 256)[1])))
                    offset = j % 2 if dt.itemsize < 16 else 0
                    assert fir_instance(dt, nb, nx, ncols, state, sms) == (dt, NT, state), (dt, nb, nx, ncols, state)
                    cases.append((dt, nb, nx, ncols, state, offset))
    return cases


def _case_id(c):
    dt, nb, nx, ncols, state, offset = c
    return f"{dt.name}-nb{nb}-nx{nx}-c{ncols}-{'state' if state else 'nostate'}-o{offset}"


CONV1_SHAPES = [(40, 9), (9, 40), (20, 20), (1, 37), (37, 1), (1, 1), (257, 255), (255, 257), (1000, 63)]
CONVN_SHAPES = [((3, 40), (5, 2)), ((5, 2), (3, 40)), ((40, 3), (2, 5)), ((3, 4), (3, 5)),
                ((4, 3, 5), (2, 6, 3)), ((2, 6, 3), (4, 3, 5)), ((3, 3, 3), (3, 2, 4)), ((6, 1, 2), (1, 5, 3))]


# =============================================================================== CPU: exact arithmetic

@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_exact_fma_against_fractions(dt):
    """fma_f32 / fma_f64 / cmuladd against one rounding of the exact value, on 10^5 triples per dtype: exponent spreads
    of +-60 (+-36 for Float32, whose exact results must stay normal), cancellations, exact and near ties, zeros.  The
    Fraction reference asserts the valid domain (no overflow, no subnormal result) at every fma."""
    dt = np.dtype(dt)
    R = _real(dt)
    rng = np.random.default_rng(1000 + DTYPES.index(dt))
    n = 100_000
    E = 36 if R == F32 else 60
    a, b, c = _triples(rng, n, R, E)
    if R == F64:                                            # fma_f64's domain: every magnitude zero or in [2^-900, 2^900]
        for t in (a, b, c, a * b):
            m = np.abs(t[t != 0])
            assert np.all((m >= 2.0 ** -900) & (m <= 2.0 ** 900))
    if not _cplx(dt):
        got = (od.fma_f32 if R == F32 else od.fma_f64)(a, b, c)
        want = np.array([_fma_q(x, y, z, R) for x, y, z in zip(a.tolist(), b.tolist(), c.tolist())], dtype=R)
        if R == F64:                                        # the data tells a fused multiply-add from an unfused one
            assert np.count_nonzero(want != a * b + c) > n // 10
    else:
        perm = rng.permutation(n)
        z = (a + 1j * b[perm]).astype(dt)
        w = (b + 1j * c[rng.permutation(n)]).astype(dt)
        x = (c + 1j * a[rng.permutation(n)]).astype(dt)
        got = od.cmuladd(z, w, x)
        want = np.array([_muladd_q(p, q, r, dt) for p, q, r in zip(z, w, x)], dtype=dt)
    assert got.dtype == want.dtype
    assert np.array_equal(got, want)


def test_exact_fma_single_cases():
    """The product's low part alone (a*b - RN(a*b)), and a sum whose Float64 rounding is a tie for the naive a*b + c:
    the exact low bits beyond it must decide, which one rounding does and two do not."""
    e = 2.0 ** -30
    a, b = 1.0 + e, 1.0 - e                                 # a*b = 1 - 2^-60
    assert od.fma_f64(a, b, -1.0) == -(2.0 ** -60) == _fma_q(a, b, -1.0, F64)
    a, b = 1.0 + 2.0 ** -26, 1.0 + 2.0 ** -27               # a*b = 1 + 3*2^-27 + 2^-53: RN(a*b) = 1 + 3*2^-27 (tie to even)
    c = 2.0 ** -80                                          # + c: just above the tie, so the fma rounds up
    assert od.fma_f64(a, b, c) == _fma_q(a, b, c, F64) == 1.0 + 3 * 2.0 ** -27 + 2.0 ** -52
    assert a * b + c == 1.0 + 3 * 2.0 ** -27
    assert od.fma_f64(3.0, -2.0, 6.0) == 0.0 and od.fma_f32(np.float32(3), np.float32(-2), np.float32(6)) == 0.0


# =============================================================================== CPU: restated chains against literal loops

@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_fir_chain_matches_literal_loop(dt):
    """The vectorised chains against the literal _filt_fir! loop with the state carried in and out: the kernel's chain
    (muladd for the last tap) and the reference's (plain product), which are the same for real eltypes."""
    dt = np.dtype(dt)
    rng = np.random.default_rng(7 + DTYPES.index(dt))
    for nb, nx in [(1, 5), (2, 7), (3, 2), (9, 20), (17, 11), (5, 1)]:
        b = _data(rng, nb, dt)
        x = _data(rng, (nx, 1), dt)
        si = _data(rng, (nb - 1, 1), dt)
        for plain in (False, True):
            y, s = fir_chain(b, x, si, state=True, plain_last=plain)
            yl, sl = fir_literal(b, x[:, 0], si[:, 0], plain)
            assert np.array_equal(y[:, 0], yl) and np.array_equal(s[:, 0], sl), (nb, nx, plain)
            y0, _ = fir_chain(b, x, None, state=False, plain_last=plain)
            yl0, _ = fir_literal(b, x[:, 0], np.zeros(nb - 1, dt), plain)
            assert np.array_equal(y0[:, 0], yl0)
    # the documented divergence: complex data, whose last tap the kernel fuses and the reference does not
    b, x = _data(rng, 9, dt), _data(rng, (200, 1), dt)
    differ = not np.array_equal(fir_chain(b, x)[0], fir_chain(b, x, plain_last=True)[0])
    assert differ == _cplx(dt)


@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_conv_chain_matches_literal_loop(dt):
    """oracle.conv_td / conv_td_nd (the reference's order, fused) against the literal _conv_td! loops, ranks 1-3, on both
    sides of the size(u,1) rule."""
    dt = np.dtype(dt)
    rng = np.random.default_rng(70 + DTYPES.index(dt))
    shapes = [((9,), (4,)), ((4,), (9,)), ((5,), (5,)), ((1,), (6,)), ((6,), (1,)), ((3, 4), (5, 2)), ((5, 2), (3, 4)),
              ((2, 3), (2, 2)), ((2, 3, 2), (3, 2, 2)), ((3, 2, 2), (2, 3, 2))]
    for su, sv in shapes:
        u, v = _data(rng, su, dt), _data(rng, sv, dt)
        want = conv_literal(u, v)
        assert np.array_equal(od.conv_td_nd(u, v), want), (su, sv)
        assert np.array_equal(conv_chain(u, v, conv_walk(u, v)), want)
        if len(su) == 1:
            assert np.array_equal(od.conv_td(u, v), want)
    # integers stay exact, and keep their dtype
    iu, iv = rng.integers(-9, 10, (7, 3)), rng.integers(-9, 10, (2, 5))
    from scipy import signal as ss
    assert np.array_equal(od.conv_td_nd(iu, iv), ss.convolve(iu, iv)) and od.conv_td_nd(iu, iv).dtype.kind == "i"
    assert np.array_equal(od.conv_td(iu[:, 0], iv[0]), np.convolve(iu[:, 0], iv[0]))


# =============================================================================== CPU: planted defects

@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_planted_fir_defects_change_the_test_data(dt):
    """Each planted defect changes at least one output bit of the true chain on the data the GPU cases use."""
    dt = np.dtype(dt)
    rng = np.random.default_rng(500 + DTYPES.index(dt))
    defects = ["reversed", "unfused", "shift", "skip_pad"] + (["swap"] if _cplx(dt) else [])
    for nb, nx in [(9, 300), (67, 300), (521, 40)]:
        b, x = _data(rng, nb, dt), _data(rng, (nx, 3), dt)
        si = _data(rng, (nb - 1, 3), dt)
        y, s = fir_chain(b, x, si, state=True)
        for d in defects:
            yd, sd = fir_chain(b, x, si, state=True, defect=d)
            assert not (np.array_equal(y, yd) and np.array_equal(s, sd)), (nb, d)


@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_planted_conv_defects_change_the_test_data(dt):
    """Reversed order, an unfused multiply-add, swapped complex operands, and the order the direct kernels used to take
    (the longer array's index ascending in 1-D, u's index always in N-D) each change an output bit; equal lengths keep
    the order, so there the old kernel agreed."""
    dt = np.dtype(dt)
    rng = np.random.default_rng(600 + DTYPES.index(dt))
    for su, sv in [((40,), (9,)), ((9,), (40,)), ((40, 3), (2, 5)), ((5, 2), (3, 40))]:
        u, v = _data(rng, su, dt), _data(rng, sv, dt)
        want = od.conv_td_nd(u, v)
        w = conv_walk(u, v)
        bad = [conv_chain(u, v, w, reverse=True), conv_chain(u, v, w, fused=False)]
        if _cplx(dt):
            bad.append(conv_chain(u, v, w, swap=True))
        if len(su) == 1:
            old = conv_chain(u, v, "u" if su[0] >= sv[0] else "v", swap=su[0] < sv[0])
        else:
            old = conv_chain(u, v, "u")
        bad.append(old)
        for i, y in enumerate(bad):
            assert not np.array_equal(y, want), (su, sv, i)
    u, v = _data(rng, (20,), dt), _data(rng, (20,), dt)
    assert np.array_equal(conv_chain(u, v, "u"), od.conv_td(u, v))


# =============================================================================== CPU: routing and case table

def test_fir_routing_restatement():
    assert fir_geom(F32, 128) == (8, 1024) and fir_geom(F64, 256) == (8, 2048) and fir_geom(C64, 256) == (8, 2048)
    assert fir_geom(C128, 128) == (4, 512) and fir_geom(C128, 256) == (4, 1024)
    assert fir_rounds(1) == [8] and fir_rounds(512) == [512] and fir_rounds(513) == [512, 8]
    assert fir_rounds(1031) == [512, 512, 8] and fir_rounds(1025) == [512, 512, 8] and fir_rounds(520) == [512, 8]
    # the 128 / 256 boundary: 8 * SMs 256-thread tiles
    assert fir_nt(F32, 2048, 8 * CPU_SMS - 1) == 128 and fir_nt(F32, 2048, 8 * CPU_SMS) == 256
    assert fir_nt(C128, 1025, 4 * CPU_SMS - 1) == 128 and fir_nt(C128, 1025, 4 * CPU_SMS) == 256
    assert fir_instance(F32, 1, 10, 1, True) == (F32, 128, False)


def _coverage(cases, sms):
    seen = {}
    for dt, nb, nx, ncols, state, offset in cases:
        inst = fir_instance(dt, nb, nx, ncols, state, sms)
        seen.setdefault(inst, set()).update(fir_features(dt, nb, nx, ncols, offset))
    return seen


def test_case_table_reaches_every_fir_instance_and_path():
    """Each of the 16 instances gets the uint4 store, a scalar tail, an unaligned column (elements below 16 bytes), a
    padding chunk and none, 1, 2 and 3 staging rounds and a kc = 8 (mod 16) tail."""
    cases = fir_cases()
    seen = _coverage(cases, CPU_SMS)
    assert set(seen) == {(dt, NT, st) for dt in DTYPES for NT in (128, 256) for st in (False, True)}
    for inst, feats in seen.items():
        assert _needed(inst[0]) <= feats, (inst, _needed(inst[0]) - feats)
    for dt in DTYPES:                                      # the suggested signal lengths, and nx < nb - 1
        nxs = {c[2] for c in cases if c[0] == dt}
        assert set(_nx_values(dt)[:4]) <= nxs and any(c[2] < c[1] - 1 for c in cases if c[0] == dt)
    assert {c[1] for c in cases} >= set(NB_128 + NB_256)
    assert {c[3] for c in cases} >= {1, 3, 70} and any(c[3] > 1000 for c in cases)


def test_conv_cases_cover_both_sides_of_the_rule():
    walks = {conv_walk(np.empty(su), np.empty(sv)) for su, sv in CONVN_SHAPES}
    assert walks == {"u", "v"} and {len(su) for su, _ in CONVN_SHAPES} == {2, 3}
    assert any(a < b for a, b in CONV1_SHAPES) and any(a > b for a, b in CONV1_SHAPES)
    assert any(a == b for a, b in CONV1_SHAPES) and any(1 in s for s in CONV1_SHAPES)
    assert all(a * b < 2 ** 16 for a, b in CONV1_SHAPES)


# =============================================================================== GPU helpers

@pytest.fixture(scope="module")
def dsp():
    return pytest.importorskip("dspb200")


def _sentinels(rng, n, dt):
    s = rng.choice(np.array([-1000.0, 1000.0]), n)
    if _cplx(dt):
        s = s + 1j * rng.choice(np.array([-1000.0, 1000.0]), n)
    return s.astype(dt)


class Guarded:
    """A device buffer of GUARD + offset cells, `n` data cells and GUARD cells: sentinels (input) or NaN (output) outside
    the data."""

    def __init__(self, dt, n, rng=None, data=None, offset=0):
        from dspb200 import device
        self.dt, self.n, self.lo = np.dtype(dt), n, GUARD + offset
        if rng is None:
            host = np.full(self.lo + n + GUARD, np.nan, dtype=dt)
        else:
            host = _sentinels(rng, self.lo + n + GUARD, dt)
        if data is not None:
            host[self.lo:self.lo + n] = np.asarray(data).ravel(order="F")
        self.host = host
        self.buf = device.to_device(host)
        self.ptr = self.buf.ptr + self.lo * self.dt.itemsize

    def data(self, shape=None):
        h = self.buf.to_host()
        outside = np.concatenate([h[:self.lo], h[self.lo + self.n:]])
        want = np.concatenate([self.host[:self.lo], self.host[self.lo + self.n:]])
        assert np.array_equal(outside, want, equal_nan=True), "a cell outside the buffer's range changed"
        d = h[self.lo:self.lo + self.n]
        return d if shape is None else d.reshape(shape, order="F")


def _device_sms(dsp):
    import ctypes as C
    sms, a, b = C.c_int(0), C.c_int(0), C.c_int(0)
    mem, l2 = C.c_size_t(0), C.c_size_t(0)
    dsp._lib.check(dsp._lib.lib.dspb200_device_info(C.byref(sms), C.byref(a), C.byref(b), C.byref(mem), C.byref(l2)))
    return sms.value


PERIOD = 7                # distinct columns of a case; the rest repeat them


def _fir_data(case):
    """(b, x, si, ref_y, ref_si): x and si are (., ncols) with columns repeating with period 7; the reference chain is
    computed on the distinct columns and tiled."""
    dt, nb, nx, ncols, state, offset = case
    rng = np.random.default_rng(zlib.crc32(_case_id(case).encode()))
    nd = min(ncols, PERIOD)
    b = _data(rng, nb, dt)
    xd = _data(rng, (nx, nd), dt)
    sd = _data(rng, (nb - 1, nd), dt)
    y, s = fir_chain(b, xd, sd if state else None, state=state)
    reps = _cdiv(ncols, nd)
    tile = (lambda a: np.asfortranarray(np.tile(a, (1, reps))[:, :ncols]))
    return b, tile(xd), tile(sd), tile(y), (tile(s) if state else None)


_FIR_CASES = fir_cases()


# =============================================================================== GPU: FIR

@pytest.mark.gpu
def test_device_routing_matches_the_case_table(dsp):
    """On this device the cases still reach every instance and path (the routing takes the device's SM count)."""
    sms = _device_sms(dsp)
    seen = _coverage(fir_cases(sms), sms)
    assert len(seen) == 16
    for inst, feats in seen.items():
        assert _needed(inst[0]) <= feats, (inst, _needed(inst[0]) - feats)


@pytest.fixture(scope="module")
def fir_cases_on_device(dsp):
    return fir_cases(_device_sms(dsp))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_fir_exec_bit_exact(dsp, fir_cases_on_device, dt):
    """dspb200_fir_exec_dev between guard cells, and the host dspb200_fir_exec, on every stateless case; the stateful
    entry points (device and host form) with a random si_in on every stateful case."""
    from dspb200 import device
    for case in (c for c in fir_cases_on_device if c[0] == dt):
        _, nb, nx, ncols, state, offset = case
        b, x, si, y, s = _fir_data(case)
        rng = np.random.default_rng(nb * 7 + nx)
        plan = dsp._lib.FirPlan(b)
        gx = Guarded(dt, nx * ncols, rng=rng, data=x, offset=offset)
        go = Guarded(dt, nx * ncols, offset=offset)
        if not state:
            plan.exec_dev(gx.ptr, nx, ncols, go.ptr, 0)
            device.sync()
            gx.data()
            assert np.array_equal(go.data((nx, ncols)), y), _case_id(case)
            out = np.empty((nx, ncols), dtype=dt, order="F")
            plan.exec(x, out)
            assert np.array_equal(out, y), _case_id(case)
        else:
            ns = nb - 1
            gsi = Guarded(dt, ns * ncols, rng=rng, data=si)
            gso = Guarded(dt, ns * ncols)
            plan.exec_state_dev(gx.ptr, nx, ncols, gsi.ptr, gso.ptr, go.ptr, 0)
            device.sync()
            gx.data(), gsi.data()
            assert np.array_equal(go.data((nx, ncols)), y), _case_id(case)
            assert np.array_equal(gso.data((ns, ncols)), s), _case_id(case)
            out = np.empty((nx, ncols), dtype=dt, order="F")
            so = np.empty((ns, ncols), dtype=dt, order="F")
            plan.exec_state(x, nx, ncols, si, so, out)
            assert np.array_equal(out, y) and np.array_equal(so, s), _case_id(case)
        plan.close()


def _front_end_cases(cases, dt, state, sms):
    """Two cases per (eltype, thread count): the first of each instance and one with more than one staging round."""
    picked = []
    for NT in (128, 256):
        mine = [c for c in cases if c[0] == dt and fir_instance(*c[:5], sms) == (dt, NT, state)]
        picked += [mine[0], next(c for c in mine if c[1] > 512)]
    return picked


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_fir_front_ends_bit_exact(dsp, fir_cases_on_device, dt):
    """filt, filt_, tdfilt on matrices, and a DF2TFilter filtering a matrix in two chunks from a random state."""
    sms = _device_sms(dsp)
    for case in _front_end_cases(fir_cases_on_device, dt, False, sms):
        b, x, _, y, _ = _fir_data(case)
        one = np.ones(1, dtype=dt)
        assert np.array_equal(dsp.filt(b, one, x), y), _case_id(case)
        out = np.empty_like(x)
        dsp.filt_(out, b, one, x)
        assert np.array_equal(out, y)
        assert np.array_equal(dsp.tdfilt(b, x), y)
    for case in _front_end_cases(fir_cases_on_device, dt, True, sms):
        nx = case[2]
        b, x, si, y, s = _fir_data(case)
        f = dsp.DF2TFilter(dsp.PolynomialRatio(b, np.ones(1, dtype=dt)), np.array(si, copy=True))
        h = nx // 2
        y1 = f.filt(np.asfortranarray(x[:h]))
        y2 = f.filt(np.asfortranarray(x[h:]))
        assert np.array_equal(np.concatenate([y1, y2]), y), _case_id(case)
        assert np.array_equal(f.state, s)


# =============================================================================== GPU: direct convolution

@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_conv_direct_1d_bit_exact(dsp, dt):
    """dspb200_conv_direct_exec, conv and conv_ (algorithm 'direct' and 'auto' below 2^16) against the reference's order;
    dspb200_conv_direct_exec bit-identical to the rank-1 dspb200_conv_nd_exec with nffts = NULL."""
    rng = np.random.default_rng(900 + DTYPES.index(dt))
    for nu, nv in CONV1_SHAPES:
        u, v = _data(rng, nu, dt), _data(rng, nv, dt)
        want = od.conv_td(u, v)
        got = np.empty(nu + nv - 1, dtype=dt)
        dsp._lib.conv_direct(u, v, got)
        assert np.array_equal(got, want), (nu, nv)
        nd = np.empty(nu + nv - 1, dtype=dt)
        dsp._lib.conv_nd(u, v, None, nd)
        assert got.tobytes() == nd.tobytes(), (nu, nv)
        for alg in ("direct", "auto"):
            assert np.array_equal(dsp.conv(u, v, algorithm=alg), want), (nu, nv, alg)
            out = np.full(nu + nv + 2, np.nan, dtype=dt)
            dsp.conv_(out, u, v, algorithm=alg)
            assert np.array_equal(out[:nu + nv - 1], want) and not np.any(out[nu + nv - 1:])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_conv_direct_nd_bit_exact(dsp, dt):
    """dspb200_conv_nd_exec and _dev with nffts = NULL, and conv (direct and auto), ranks 2 and 3, both sides of the
    size(u,1) rule; the device form between guard cells."""
    from dspb200 import device
    rng = np.random.default_rng(950 + DTYPES.index(dt))
    for su, sv in CONVN_SHAPES:
        u, v = _data(rng, su, dt), _data(rng, sv, dt)
        want = od.conv_td_nd(u, v)
        so = want.shape
        uF, vF = np.asfortranarray(u), np.asfortranarray(v)
        got = np.empty(so, dtype=dt, order="F")
        dsp._lib.conv_nd(uF, vF, None, got)
        assert np.array_equal(got, want), (su, sv)
        gu = Guarded(dt, u.size, rng=rng, data=uF)
        gv = Guarded(dt, v.size, rng=rng, data=vF)
        go = Guarded(dt, want.size)
        dsp._lib.conv_nd_dev(dt, su, gu.ptr, sv, gv.ptr, None, go.ptr)
        device.sync()
        gu.data(), gv.data()
        assert np.array_equal(go.data(so), want), (su, sv)
        for alg in ("direct", "auto"):
            assert np.array_equal(dsp.conv(u, v, algorithm=alg), want), (su, sv, alg)
