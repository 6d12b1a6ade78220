"""Every instance and entry point of the arbitrary-rate resampler (resample_arb_batch_kernel, csrc/resample.cu) against
exact rational phases, output by output.

The kernel runs in six (input, taps) type combinations, each with and without HIST (the streaming form that reads the
virtual column [history; chunk]): 12 instances.  It is reached through exec(_dev), batch_exec(_dev) and
stream_exec_dev.  Output j of a call sits at total phase P_j = acc0 + j*delta, which `ExactPhase` evaluates exactly
from the two doubles as scaled Python integers: s = floor(P_j) (phase index q*N + phi), and the fraction alpha.

The phase bound.  With u = 2^-53 and N = nphases, the kernel's phase (arb_phase) is within BETA = C_PHASE * u * N
phases of the exact one.  The C ABI refuses acc0 outside [0, N), so N bounds every term of the phase sum: r = fma(-q,
N, hi) is exact, then (r + lo) + acc0 rounds twice on values below 2N and the `while` correction once more on values
below N, at most 4 u N together.  `test_arb_phase_restated_within_bound` shows the restated arb_phase inside that
bound over every N, acc0 and delta of interest, with j up to 2^53 / delta (the largest error seen is u N, at N = 1).
When the exact phase is farther than BETA from every integer the output must use (q*, phi*); otherwise either
neighbouring (q, phi) is accepted, with alpha near 0 or near 1 (the derivative bank ends each row with diff(h) = 0 at
the wrap, so the two branches differ there: both are computed).

Integer data.  Taps are integers in [-4, 4] and samples integers in [-8, 8] (both parts for complex data), so both dot
products yl and yu are exact integers in every type combination, and each output must satisfy
    |y - (yu * alpha* + yl)| <= |yu| * BETA + 1/2 ulp_EO(y*)      (+ 2^-53 |y*| for the double-then-Float32 rounding)
component by component: a Float32 output within half an ulp of the exact value, a Float64 output within the phase
bound.  Random data (Gaussian samples, resample_filter taps) gets the per-output bound
    gamma_tpp(u_EO) * (sum|pfb||x| + |alpha| sum|dpfb||x|) + |yu| * BETA + 1/2 ulp
against a long-double reference at the exact phase.

Inputs sit between sentinel samples of magnitude 1000 (in front, by a base offset, and behind, in the rows ldx > nx of
every column), so one read outside [0, nx) changes an integer output; outputs and stream histories sit between NaN
cells that must survive every call.  `test_checker_rejects_planted_defects` runs a numpy model of the kernel with each
of seven defects and shows the checker refuses every one; `test_case_table_reaches_every_regime` restates
rs_arb_tiling and the vec16 rule and shows the GPU case table reaches each instance and regime."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import filters as of
from oracle.dspbase import fma_f64

F32, F64, C64, C128 = (np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))
# the six (input, taps) combinations that select distinct instances in rs_with_types (resample.cu)
TRIPLES = ((F32, F32), (F32, F64), (F64, F64), (C64, F32), (C64, F64), (C128, F64))
TRIPLE_IDS = [f"{a}-{b}" for a, b in TRIPLES]
RATES = (0.98, 1.0001, 1.2957, 2.618, 0.7312, 1 / 55.55)
SMEM_OPTIN = 227 * 1024          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
SPAN_MAX = BANKS_MAX = 96 * 1024  # RS_ARB_SPAN_MAX, RS_ARB_BANKS_MAX
U = 2.0 ** -53
C_PHASE = 4.0
GUARD = 64                       # sentinel / NaN cells on each side of a device buffer
LD = np.longdouble
LDC = np.clongdouble


def beta(N):
    """Phase bound of arb_phase, in phases."""
    return C_PHASE * U * N


def out_dtype(dx, dh):
    """promote_type(eltype(h), eltype(x)) as the plan reports it (Float64 taps make Float64 arithmetic)."""
    return np.result_type(np.dtype(dx), np.dtype(dh))


def _real(dt):
    return np.dtype(dt).type(0).real.dtype


def _cplx(dt):
    return np.dtype(dt).kind == "c"


# =============================================================================== exact phases

class ExactPhase:
    """P_j = acc0 + j*delta for the doubles acc0 and delta, exactly: both are integers over a common power of two L."""

    def __init__(self, acc0, delta, N):
        a, da = float(acc0).as_integer_ratio()
        d, dd = float(delta).as_integer_ratio()
        self.L = max(da, dd)
        self.A, self.D, self.N = a * (self.L // da), d * (self.L // dd), int(N)
        self.acc0, self.delta = float(acc0), float(delta)

    def at(self, js):
        """(s, ahi, alo, side) per j: s = floor(P_j) as int64, alpha* = ahi + alo (to ~2^-106), side = -1 when P_j lies
        within BETA above s, +1 when within BETA below s + 1, else 0."""
        L, A, D = self.L, self.A, self.D
        lim = beta(self.N) * L
        n = len(js)
        s = np.empty(n, dtype=np.int64)
        ahi, alo = np.empty(n), np.empty(n)
        side = np.zeros(n, dtype=np.int64)
        for k, j in enumerate(np.asarray(js).tolist()):
            fl, fr = divmod(A + j * D, L)
            s[k] = fl
            hi = fr / L                                         # correctly rounded
            hn, hd = hi.as_integer_ratio()
            ahi[k] = hi
            alo[k] = (fr * hd - hn * L) / (L * hd)
            if fr <= lim:
                side[k] = -1
            elif L - fr <= lim:
                side[k] = 1
        return s, ahi, alo, side

    def q_exact(self, js):
        NL = self.N * self.L
        return np.array([(self.A + j * self.D) // NL for j in np.asarray(js).tolist()], dtype=np.int64)


# =============================================================================== arb_phase restated

def arb_phase_model(js, N, acc0, delta, contract=False, naive=False, no_while=False):
    """arb_phase (resample.cu) in numpy doubles.  contract: `hi + acc0` fused into fma(j, delta, acc0), as nvcc may do.
    naive / no_while: planted defects (P as acc0 + j*delta in one double; no `while` correction)."""
    jd = np.asarray(js, dtype=np.float64)
    N = float(N)
    acc = np.full_like(jd, acc0)
    if naive:
        P = acc0 + jd * delta
        q = np.floor(P / N)
        return q, P - q * N
    hi = jd * delta
    lo = fma_f64(jd, np.full_like(jd, delta), -hi)
    s = fma_f64(jd, np.full_like(jd, delta), acc) if contract else hi + acc
    q = np.floor(s / N)
    r = fma_f64(-q, np.full_like(jd, N), hi)
    r = (r + lo) + acc0
    if not no_while:
        for _ in range(8):
            neg = r < 0.0
            r, q = np.where(neg, r + N, r), np.where(neg, q - 1.0, q)
            big = r >= N
            r, q = np.where(big, r - N, r), np.where(big, q + 1.0, q)
            if not (neg.any() or big.any()):
                break
        assert not ((r < 0.0) | (r >= N)).any()
    return q, r


# =============================================================================== tiling restated from rs_arb_tiling

def arb_tiling(tpp, nphi, delta, x_bytes, tap_bytes):
    """(tile, threads, xs_len, banks_in_smem, smem bytes) as rs_arb_tiling computes them."""
    bank_bytes = 2 * nphi * tpp * tap_bytes
    banks = bank_bytes <= BANKS_MAX
    V = 16 // x_bytes
    tile, xs_len = 256, 0
    for T in (1024, 512, 256, 128, 64, 32):
        steps = math.ceil((T - 1) * delta / nphi)
        if steps * x_bytes > SPAN_MAX:
            continue
        span = steps + tpp + 1
        n = (span + V - 1 + V - 1) // V * V
        if n * x_bytes > SPAN_MAX:
            continue
        tile, xs_len = T, n
        break
    return tile, min(tile, 256), xs_len, banks, xs_len * x_bytes + (bank_bytes if banks else 0)


def _tr_bytes(dx, dh):
    return 8 if np.dtype(dx) in (F64, C128) or np.dtype(dh) == F64 else 4


def vec16(base_offset_elems, ldx, x_bytes):
    """rs_arb_launch: 16-byte copies when the column base is 16-byte aligned and so is the column stride (device
    buffers are 256-byte aligned, so the base's alignment is that of its element offset)."""
    return (base_offset_elems * x_bytes) % 16 == 0 and (ldx * x_bytes) % 16 == 0


def banks(h, N):
    """(pfb, dpfb) as float64 tpp x N matrices: taps2pfb(h) and taps2pfb([diff(h); 0]), the difference in the taps'
    own precision as the plan computes it."""
    h = np.asarray(h)
    dh = np.concatenate([np.diff(h), np.zeros(1, dtype=h.dtype)])
    return of.taps2pfb(h.astype(np.float64), N), of.taps2pfb(dh.astype(np.float64), N)


# =============================================================================== reference and checker

def _gather(X, idx):
    """Rows idx of the columns X (L x ncols), zero outside [0, L), as long double."""
    L = X.shape[0]
    ok = (idx >= 0) & (idx < L)
    v = X[np.clip(idx, 0, max(L - 1, 0))] if L else np.zeros((len(idx), X.shape[1]), dtype=X.dtype)
    v = np.where(ok[:, None], v, 0)
    return v.astype(LDC if _cplx(X.dtype) else LD)


def _branch(X, pfb, dpfb, n0, N, s_b):
    """yl, yu and sum|pfb||x|, sum|dpfb||x| per component, for phase index s_b (int64): long double."""
    tpp = pfb.shape[0]
    q, phi = s_b // N, s_b % N
    first = n0 + q - (tpp - 1)
    cplx = _cplx(X.dtype)
    shape = (len(s_b), X.shape[1])
    yl = np.zeros(shape, dtype=LDC if cplx else LD)
    yu = np.zeros_like(yl)
    sl = [np.zeros(shape, dtype=LD) for _ in range(2)]
    su = [np.zeros(shape, dtype=LD) for _ in range(2)]
    for t in range(tpp):
        v = _gather(X, first + t)
        hl = pfb[t, phi].astype(LD)[:, None]
        hu = dpfb[t, phi].astype(LD)[:, None]
        yl += hl * v
        yu += hu * v
        for c, part in enumerate((v.real, v.imag) if cplx else (v,)):
            sl[c] += np.abs(hl) * np.abs(part)
            su[c] += np.abs(hu) * np.abs(part)
    return yl, yu, sl, su


def _half_ulp(m, eo):
    """Half an ulp of the real type eo at magnitude m (>= 0), from the binade of m."""
    p = np.finfo(eo).nmant + 1
    _, e = np.frexp(np.asarray(m, dtype=np.float64))
    return np.ldexp(np.ones_like(m, dtype=np.float64), e - p - 1)


def check_outputs(y, X, pfb, dpfb, n0, ph, js, exact_data, what=""):
    """Outputs y (len(js) x ncols, the kernel's element type) of columns X (zero outside [0, len(X))) at outputs js
    against the exact phase `ph`, within the per-output bound.  Returns the largest error-to-bound ratio."""
    if len(js) == 0:
        return 0.0
    y = np.asarray(y).reshape(len(js), -1)
    eo = _real(y.dtype)
    N = ph.N
    B = beta(N)
    tpp = pfb.shape[0]
    uo = np.finfo(eo).eps / 2
    gam = 0.0 if exact_data else tpp * uo / (1 - tpp * uo)
    s, ahi, alo, side = ph.at(js)
    cplx = _cplx(y.dtype)
    comps_y = (y.real, y.imag) if cplx else (y,)
    best = None                                                   # per output: smallest ratio over accepted branches
    for off in (0, -1, 1):
        use = side == off if off else np.ones(len(js), dtype=bool)
        if off and not use.any():
            continue
        s_b = s + off
        alpha = (ahi.astype(LD) + alo.astype(LD) - off)[:, None]
        yl, yu, sl, su = _branch(X, pfb, dpfb, n0, N, s_b)
        ratio = np.zeros(y.shape, dtype=np.float64)
        for c, yc in enumerate(comps_y):
            l, u_ = (yl.real, yu.real) if c == 0 else (yl.imag, yu.imag)
            if not cplx:
                l, u_ = yl, yu
            want = u_ * alpha + l
            aw = np.abs(want)
            rest = gam * (sl[c] + np.abs(alpha) * su[c]) + (np.abs(u_) + gam * su[c]) * B * (1 + 2.0 ** -20)
            rest += (np.abs(l) + np.abs(u_)) * 2.0 ** -60              # the long-double reference's own rounding
            m = (aw + rest).astype(np.float64) * (1 + 2.0 ** -40)
            bound = rest.astype(np.float64) + _half_ulp(m, eo) + (U * m if eo == np.float32 else 0.0)
            err = np.abs(yc.astype(LD) - want).astype(np.float64)
            r = np.where(err <= bound, err / np.maximum(bound, 1e-300), np.inf)
            r = np.where(np.isnan(yc), np.inf, r)
            ratio = np.maximum(ratio, r)
        ratio[~use] = np.inf
        best = ratio if best is None else np.minimum(best, ratio)
    bad = np.argwhere(~(best <= 1.0))
    assert bad.size == 0, (f"{what}: {len(bad)} outputs outside the bound, first (probe, column) "
                           f"{[(int(js[i]), int(c)) for i, c in bad[:4]]}")
    return float(best.max()) if best.size else 0.0


# =============================================================================== CPU: arb_phase within the bound

def _acc0_values(N):
    vals = {0.0, math.nextafter(float(N), 0.0), 2.0 ** -60}
    so = of.FIRArbitraryState(np.ones(12 * N - 5), 0.98, N)      # undelay! of a 12-taps-per-phase filter
    so.setphase(so.timedelay())
    vals.add(so.acc)
    for k in sorted({1, N // 2, N - 1}):
        if 1 <= k < N:
            vals |= {math.nextafter(float(k), 0.0), k - 2.0 ** -30, math.nextafter(float(k), math.inf), k + 2.0 ** -30}
    vals.add(N * 0.6180339887498949)
    return sorted(v for v in vals if 0.0 <= v < N)


def _deltas(N):
    return sorted({N / r for r in RATES} | {1.0, 3.0, float(N + 1), float(2 * N - 1), float(N)})


def _phase_errors(N, acc0, delta, js, **kw):
    """(worst |P_model - P*| in units of u*N, q wrong where it must be right, r out of [0, N))."""
    q, r = arb_phase_model(js, N, acc0, delta, **kw)
    ph = ExactPhase(acc0, delta, N)
    L, B = ph.L, beta(N)
    worst, qbad = 0.0, 0
    qx = ph.q_exact(js)
    for k, j in enumerate(np.asarray(js).tolist()):
        rn, rd = float(r[k]).as_integer_ratio()
        assert L % rd == 0
        e = int(q[k]) * N * L + rn * (L // rd) - (ph.A + j * ph.D)
        worst = max(worst, abs(e) / L / (U * N))
        rx = (ph.A + j * ph.D) - int(qx[k]) * N * L                # exact r* * L
        if int(q[k]) != int(qx[k]) and B * L < rx < N * L - B * L:
            qbad += 1
    return worst, qbad, int(((r < 0) | (r >= N)).sum())


@pytest.mark.parametrize("N", [1, 3, 7, 32, 100, 128, 1024])
def test_arb_phase_restated_within_bound(N):
    rng = np.random.default_rng(N)
    worst = 0.0
    for acc0 in _acc0_values(N):
        for delta in _deltas(N):
            # j and the whole phase acc0 + j*delta (so q) stay below 2^53, where doubles hold every integer
            jmax = min(int((2.0 ** 53 - 2 * N) / delta), 2 ** 53)
            js = np.unique(np.concatenate([
                np.arange(0, 64), jmax - np.arange(0, 16),
                np.exp(rng.uniform(0, math.log(jmax), 160)).astype(np.int64),
                (2 ** np.arange(10, 53)) // max(1, int(delta))]))
            js = js[(js >= 0) & (js <= jmax)]
            for contract in (False, True):
                w, qbad, rbad = _phase_errors(N, acc0, delta, js, contract=contract)
                assert qbad == 0 and rbad == 0, (N, acc0, delta, contract)
                worst = max(worst, w)
    print(f"N = {N}: worst restated arb_phase error {worst:.3f} u N (bound {C_PHASE} u N)")
    assert worst <= C_PHASE


def test_naive_phase_leaves_the_bound():
    """The phase bound is tight enough to tell the split product from acc0 + j*delta in one double at j*delta ~ 2^31."""
    js = np.arange(2 ** 26, 2 ** 26 + 256)
    w, _, _ = _phase_errors(32, 0.3 * 32, 32 / 0.98, js, naive=True)
    assert w > 1000 * C_PHASE


# =============================================================================== CPU: numpy model of the kernel, planted defects

DEFECTS = ("alpha_f32", "naive_phase", "no_while", "window_shift", "drow_next", "span_tap", "tile_last_unwritten")


def model_kernel(X, pfb, dpfb, N, n0, acc0, delta, js, eo_dtype, tile, defect=None):
    """The kernel's outputs at js for columns X (exact integer data: the dot products are exact in any order)."""
    tpp = pfb.shape[0]
    q, r = arb_phase_model(js, N, acc0, delta, naive=defect == "naive_phase", no_while=defect == "no_while")
    fl = np.floor(r)
    phi = fl.astype(np.int64) % N                                  # no_while: a row index of -1 or N wraps
    alpha = r - fl
    if defect == "alpha_f32":
        alpha = alpha.astype(np.float32).astype(np.float64)
    first = n0 + q.astype(np.int64) - (tpp - 1) + (1 if defect == "window_shift" else 0)
    drow = (phi + 1) % N if defect == "drow_next" else phi
    cplx = _cplx(X.dtype)

    def dots(Xs):
        yl = np.zeros((len(js), X.shape[1]), dtype=np.complex128 if cplx else np.float64)
        yu = np.zeros_like(yl)
        for t in range(tpp):
            idx = first + t
            ok = (idx >= 0) & (idx < Xs.shape[0])
            v = np.where(ok[:, None], Xs[np.clip(idx, 0, Xs.shape[0] - 1)], 0)
            yl += pfb[t, phi][:, None] * v
            yu += dpfb[t, drow][:, None] * v
        return yl, yu

    yl, yu = dots(X)
    k = 2                                                          # the tile a tile-local defect hits
    in_tile = (np.asarray(js) >= k * tile) & (np.asarray(js) < (k + 1) * tile)
    if defect == "span_tap":
        # one staged sample of tile k's span holds a wrong value: the newest sample of the tile's first output
        s0 = int(first[np.argmax(in_tile)]) + tpp - 1
        Xb = X.copy()
        Xb[s0] += 1
        yl2, yu2 = dots(Xb)
        yl, yu = np.where(in_tile[:, None], yl2, yl), np.where(in_tile[:, None], yu2, yu)
    a = alpha[:, None]

    def mix(u_, l):
        return fma_f64(u_, np.broadcast_to(a, u_.shape), l)

    y = (mix(yu.real, yl.real) + 1j * mix(yu.imag, yl.imag)) if cplx else mix(yu, yl)
    y = y.astype(eo_dtype)
    if defect == "tile_last_unwritten":
        y[np.asarray(js) == (k + 1) * tile - 1] = np.nan
    return y


def _model_case(dx, dh, seed, N=32, rate=0.98, big_j=False):
    """Integer column, taps and the exact-phase arguments of one model run; big_j: outputs around j = 2^26 of a short
    column (a negative n0 puts their windows inside it)."""
    rng = np.random.default_rng(seed)
    hlen = 12 * N - 5
    h = rng.integers(-4, 5, hlen).astype(dh)
    pfb, dpfb = banks(h, N)
    tpp = pfb.shape[0]
    so = of.FIRArbitraryState(np.ones(hlen), rate, N)
    so.setphase(so.timedelay())
    acc0, delta = so.acc, N / rate
    j0 = 2 ** 26 if big_j else 0
    js = np.arange(j0, j0 + 4096)
    n0 = 3 - int(ExactPhase(acc0, delta, N).q_exact([j0])[0]) if big_j else 3
    nx = int(4096 * delta / N) + 8
    X = int_signal(rng, (nx, 2), dx)
    tile = arb_tiling(tpp, N, delta, np.dtype(dx).itemsize, _tr_bytes(dx, dh))[0]
    return X, pfb, dpfb, N, n0, acc0, delta, js, tile


def _rejects(X, pfb, dpfb, N, n0, acc0, delta, js, eo, tile, defect):
    y = model_kernel(X, pfb, dpfb, N, n0, acc0, delta, js, eo, tile, defect)
    try:
        check_outputs(y, X, pfb, dpfb, n0, ExactPhase(acc0, delta, N), js, True, defect)
    except AssertionError:
        return True
    return False


@pytest.mark.parametrize("dx,dh", [(F32, F32), (F64, F64), (C64, F32)], ids=str)
def test_checker_rejects_planted_defects(dx, dh):
    eo = out_dtype(dx, dh)
    for big_j in (False, True):
        args = _model_case(dx, dh, 5, big_j=big_j)
        X, pfb, dpfb, N, n0, acc0, delta, js, tile = args
        y = model_kernel(*args[:8], eo, tile)
        check_outputs(y, X, pfb, dpfb, n0, ExactPhase(acc0, delta, N), js, True, "clean model")
    # each defect on the run where it shows: the naive phase at j*delta ~ 2^31, no_while below, the rest at small j
    small, big = _model_case(dx, dh, 6), _model_case(dx, dh, 7, big_j=True)
    for defect in DEFECTS:
        if defect == "no_while":
            continue
        assert _rejects(*(big if defect == "naive_phase" else small)[:8], eo, small[8], defect), defect
    # no_while needs a phase that the first estimate puts one N too far: acc0 just below N and an integer delta
    X, pfb, dpfb, N, _, _, _, _, tile = small
    acc0, delta = 32 - 2.0 ** -40, 3.0
    js = np.arange(20000, 20000 + 2048)
    n0 = 5 - int(ExactPhase(acc0, delta, N).q_exact([20000])[0])
    assert _rejects(X, pfb, dpfb, N, n0, acc0, delta, js, eo, tile, "no_while")
    y = model_kernel(X, pfb, dpfb, N, n0, acc0, delta, js, eo, tile)
    check_outputs(y, X, pfb, dpfb, n0, ExactPhase(acc0, delta, N), js, True, "clean model, corrected phases")
    print(f"{dx}-{dh}: every planted defect rejected: {', '.join(DEFECTS)}")


# =============================================================================== the case table

def int_taps(rng, hlen, dt):
    return rng.integers(-4, 5, hlen).astype(dt)


def int_signal(rng, shape, dt):
    v = rng.integers(-8, 9, shape).astype(np.float64)
    if np.dtype(dt).kind == "c":
        v = v + 1j * rng.integers(-8, 9, shape)
    return v.astype(dt)


def _undelay_acc(hlen, rate, N):
    so = of.FIRArbitraryState(np.ones(hlen), rate, N)
    so.setphase(so.timedelay())
    return so.acc


def one_shot_cases():
    """Calls of the non-HIST instances: dict(dx, dh, N, hlen, delta, acc0, n0, nx, ldx, ncols, nout, offset, entry)."""
    cases = []
    for dx, dh in TRIPLES:
        V = 16 // dx.itemsize
        base = dict(dx=dx, dh=dh)
        # N = 32, 12 taps per phase, non-dyadic rates with undelay! phases; windows straddle both ends
        for k, rate in enumerate((0.98, 1.2957, 2.618)):
            delta = 32 / rate
            nout = 3000
            nx = int(nout * delta / 32) - 4
            cases.append(dict(base, N=32, hlen=12 * 32 - 5, delta=delta, acc0=_undelay_acc(12 * 32 - 5, rate, 32), n0=2,
                              nx=nx, ldx=nx + 2 * V, ncols=3, nout=nout, offset=0, entry="batch_dev"))
        cases.append(dict(base, N=32, hlen=12 * 32 - 5, delta=32 / 0.7312, acc0=17.123456789, n0=9, nx=2001, ldx=2003,
                          ncols=70, nout=1400, offset=1, entry="batch_dev"))
        cases.append(dict(base, N=32, hlen=12 * 32 - 5, delta=32 / 0.98, acc0=0.6180339887498949 * 32, n0=4, nx=3000,
                          ldx=3000, ncols=1, nout=2900, offset=0, entry="exec_dev"))
        cases.append(dict(base, N=32, hlen=12 * 32 - 5, delta=32 / 0.98, acc0=0.6180339887498949 * 32, n0=4, nx=3000,
                          ldx=3000, ncols=1, nout=2900, offset=3, entry="exec_dev"))
        # N not a power of two, interpolating; N = 100 decimating by 55.55 (small tiles for wide types)
        cases.append(dict(base, N=7, hlen=7 * 9, delta=7 / 2.618, acc0=_undelay_acc(63, 2.618, 7), n0=1, nx=1500, ldx=1500,
                          ncols=3, nout=4000, offset=0, entry="batch_dev"))
        cases.append(dict(base, N=100, hlen=100 * 5, delta=100 * 55.55, acc0=_undelay_acc(500, 1 / 55.55, 100), n0=3,
                          nx=60000, ldx=60001, ncols=2, nout=1100, offset=0, entry="batch_dev"))
        # xs_len = 0: the span of 32 outputs is over 96 KB
        cases.append(dict(base, N=32, hlen=12 * 32 - 5, delta=32 * 1000.0 + 0.37, acc0=31.25, n0=1, nx=150000,
                          ldx=150000, ncols=2, nout=160, offset=0, entry="batch_dev"))
        # banks in global memory: 400 taps per phase
        cases.append(dict(base, N=32, hlen=400 * 32, delta=32 / 1.2957, acc0=_undelay_acc(400 * 32, 1.2957, 32), n0=30,
                          nx=2500, ldx=2500, ncols=2, nout=3400, offset=0, entry="batch_dev"))
        # tpp = 1; N = 1; an integer delta with acc0 just below N (phases on and beside the boundaries)
        cases.append(dict(base, N=32, hlen=20, delta=32 / 0.7312, acc0=math.nextafter(32.0, 0.0), n0=0, nx=800,
                          ldx=800, ncols=2, nout=1100, offset=0, entry="batch_dev"))
        cases.append(dict(base, N=1, hlen=21, delta=1 / 0.7312, acc0=0.4321, n0=0, nx=1000, ldx=1000, ncols=2,
                          nout=1390, offset=0, entry="batch_dev"))
        cases.append(dict(base, N=32, hlen=8 * 32, delta=33.0, acc0=32 - 2.0 ** -40, n0=0, nx=20700, ldx=20700, ncols=1,
                          nout=20000, offset=0, entry="batch_dev"))
        cases.append(dict(base, N=32, hlen=8 * 32, delta=32.0, acc0=2.0 ** -44, n0=0, nx=3000, ldx=3000, ncols=1,
                          nout=3000, offset=0, entry="batch_dev"))
    # more columns than one grid dimension holds
    for dx, dh in ((F32, F32), (C64, F64)):
        cases.append(dict(dx=dx, dh=dh, N=32, hlen=3 * 32, delta=32 / 0.98, acc0=5.5, n0=1, nx=7, ldx=7, ncols=70000,
                          nout=6, offset=0, entry="batch_dev"))
    return cases


def stream_chains():
    """Chunk sequences of the HIST instances: one FIRArbitrary state carried through the chunk sizes (0: a NULL
    history), with `ncols` channels."""
    chains = []
    for dx, dh in TRIPLES:
        chains.append(dict(dx=dx, dh=dh, N=32, hlen=12 * 32 - 5, rate=0.98, ncols=3, chunks=(1000, 5, 999, 1, 3, 2048, 7)))
        chains.append(dict(dx=dx, dh=dh, N=7, hlen=7 * 6, rate=2.618, ncols=2, chunks=(300, 4, 301)))
        chains.append(dict(dx=dx, dh=dh, N=32, hlen=20, rate=1.2957, ncols=2, chunks=(50, 1, 64)))      # tpp = 1: H = 0
    return chains


def _case_regimes(c):
    """Regimes one non-HIST call reaches, from the restated tiling and exact phases."""
    dx, N = c["dx"], c["N"]
    tpp = -(-c["hlen"] // N)
    xb = dx.itemsize
    V = 16 // xb
    tile, threads, xs_len, bk, smem = arb_tiling(tpp, N, c["delta"], xb, _tr_bytes(dx, c["dh"]))
    assert smem <= SMEM_OPTIN
    out = {f"instance {dx}-{c['dh']} plain", "banks in shared memory" if bk else "banks in global memory"}
    v16 = vec16(c["offset"], c["ldx"], xb)
    out.add("xs_len = 0" if xs_len == 0 else f"staged span, {'with' if v16 else 'without'} vec16")
    out |= {"tile < 256"} if tile < 256 else set()
    out |= _window_regimes(c["acc0"], c["delta"], N, tpp, c["n0"], c["nx"], c["nout"], tile, xs_len, V, 0)
    if tpp == 1:
        out.add("tpp = 1")
    if N == 1:
        out.add("N = 1")
    if N & (N - 1):
        out.add("N not a power of two")
    return out


def _window_regimes(acc0, delta, N, tpp, n0, ncol, nout, tile, xs_len, V, hlen):
    out = set()
    js = np.arange(nout)
    q = ExactPhase(acc0, delta, N).q_exact(js)
    first = n0 + q - (tpp - 1)
    if xs_len:
        gb = first[(js // tile) * tile]                          # the span start of each output's tile
        xb = gb - ((gb - hlen) % V)
        inside = (first >= xb) & (first + tpp <= xb + xs_len)
    else:
        inside = np.zeros(nout, dtype=bool)
    if inside.any():
        out.add("windows inside the span")
    if (~inside).any():
        out.add("windows by the global bounds test")
    if ((first < 0) & (first + tpp > 0)).any():
        out.add("window straddles sample 0")
    if ((first < ncol) & (first + tpp > ncol)).any():
        out.add("window straddles sample nx")
    return out


def _chain_calls(ch):
    """(nx, input_deficit, acc0, n0, nout, NULL history?) per chunk, from the FIRFilter bookkeeping."""
    import dspb200 as dsp
    f = dsp.FIRFilter(np.ones(ch["hlen"]), ch["rate"], ch["N"])
    f.setphase(f.timedelay())
    calls = []
    for k, nx in enumerate(ch["chunks"]):
        st = f._step(f.phi_idx, f.input_deficit, f.phi_accumulator, nx)
        calls.append((nx, f.input_deficit, st.phase0, st.n0, st.nout, k == 0))
        f._commit(st)
    return calls, f.delta


def _chain_regimes(ch):
    dx, N = ch["dx"], ch["N"]
    tpp = -(-ch["hlen"] // N)
    H = tpp - 1
    xb = dx.itemsize
    V = 16 // xb
    calls, delta = _chain_calls(ch)
    out = {f"instance {dx}-{ch['dh']} HIST"}
    tile, _, xs_len, bk, _ = arb_tiling(tpp, N, delta, xb, _tr_bytes(dx, ch["dh"]))
    for nx, _, acc0, n0, nout, null in calls:
        if nout == 0:
            continue
        if null:
            out.add("NULL history")
        if nx < H:
            out.add("chunk shorter than the history")
        if xs_len and vec16(0, nx, xb) and H % V:
            out.add("history/chunk seam inside a 16-byte vector")
        out |= _window_regimes(acc0, delta, N, tpp, n0, H + nx, nout, tile, xs_len, V, H)
    if tpp == 1:
        out.add("tpp = 1")
    return out


REQUIRED = ({f"instance {a}-{b} {k}" for a, b in TRIPLES for k in ("plain", "HIST")}
            | {"staged span, with vec16", "staged span, without vec16", "xs_len = 0", "banks in shared memory",
               "banks in global memory", "tile < 256", "windows inside the span", "windows by the global bounds test",
               "window straddles sample 0", "window straddles sample nx", "NULL history", "chunk shorter than the history",
               "history/chunk seam inside a 16-byte vector", "tpp = 1", "N = 1", "N not a power of two"})


def test_case_table_reaches_every_regime():
    seen = set()
    for c in one_shot_cases():
        seen |= _case_regimes(c)
    for ch in stream_chains():
        seen |= _chain_regimes(ch)
    print("regimes reached:\n  " + "\n  ".join(sorted(seen)))
    assert REQUIRED <= seen, sorted(REQUIRED - seen)


# =============================================================================== CPU: the streaming phase state

def test_stream_state_rounds_once_per_chunk():
    """_arb_advance: each chunk's acc0 is the correctly rounded exact phase after the previous chunk (from that chunk's
    own double acc0), and the phase of the whole concatenation drifts by at most half an ulp of N per chunk."""
    from dspb200.filters import _arb_advance
    rng = np.random.default_rng(3)
    for N, rate in ((32, 0.98), (32, 2.618), (32, 1 / 55.55), (64, 1.0001)):
        delta = N / rate
        acc, deficit = _undelay_acc(12 * N - 5, rate, N), 4
        G0 = Fraction(deficit - 1) * N + Fraction(acc)            # total phase of the stream's first output
        consumed, total_out = 0, 0
        for k in range(400):
            xlen = int(rng.choice([1, 2, 10, 11, int(rng.integers(1, 5000))]))
            if xlen < deficit:
                deficit -= xlen
                consumed += xlen
                continue
            nout, new_deficit, new_acc = _arb_advance(acc, deficit, delta, N, xlen)
            P = Fraction(acc) + nout * Fraction(delta)
            q = P // N
            want = float(P - q * N)
            if want >= N:
                want = math.nextafter(float(N), 0.0)
            assert new_acc == want and new_deficit == deficit + int(q) - xlen
            consumed += xlen
            total_out += nout
            acc, deficit = new_acc, new_deficit
            G = Fraction(consumed + deficit - 1) * N + Fraction(acc)
            exact = G0 + total_out * Fraction(delta)
            assert abs(G - exact) <= (k + 1) * Fraction(math.ulp(float(N))) / 2, (N, rate, k)


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
    """A device buffer of GUARD cells, `n` data cells (from `offset` cells on) and GUARD cells: sentinels (input) or NaN
    (output) outside the data."""

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
        """The data cells (Fortran-ordered `shape`), after checking that the cells around them are unchanged."""
        h = self.buf.to_host()
        outside = np.concatenate([h[:self.lo], h[self.lo + self.n:]])
        want = np.concatenate([self.host[:self.lo], self.host[self.lo + self.n:]])
        assert np.array_equal(outside, want, equal_nan=True), "a cell outside the buffer's range changed"
        d = h[self.lo:self.lo + self.n]
        return d if shape is None else d.reshape(shape, order="F")


_RATIOS = {}


def _note(dx, dh, hist, ratio):
    """Record a ratio under the instance rs_with_types picks: Float64 and ComplexF64 input always run Float64 taps."""
    dx, dh = np.dtype(dx), np.dtype(dh)
    if dx in (F64, C128):
        dh = F64
    key = f"{dx}-{dh} {'HIST' if hist else 'plain'}"
    _RATIOS[key] = max(_RATIOS.get(key, 0.0), ratio)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8)


def _run_one_shot(dsp, c, seed):
    """One case through its device entry point with guard cells, and through the matching host entry point; both
    checked against the exact phases, and bit-equal."""
    from dspb200 import device
    rng = np.random.default_rng(seed)
    dx, dh, N, nx, ldx, ncols, nout = c["dx"], c["dh"], c["N"], c["nx"], c["ldx"], c["ncols"], c["nout"]
    h = int_taps(rng, c["hlen"], dh)
    pfb, dpfb = banks(h, N)
    X = int_signal(rng, (ldx, ncols), dx)
    X[nx:] = _sentinels(rng, (ldx - nx) * ncols, dx).reshape(ldx - nx, ncols)   # rows the kernel must not read
    plan = dsp._lib.ResampleArbPlan(dx, h, N)
    eo = plan.out_dtype
    assert eo == out_dtype(dx, dh)
    gx = Guarded(dx, ldx * ncols, rng=rng, data=X, offset=c["offset"])
    go = Guarded(eo, nout * ncols)
    if c["entry"] == "exec_dev":
        assert ncols == 1 and ldx == nx
        plan.exec_dev(gx.ptr, nx, c["n0"], c["acc0"], c["delta"], go.ptr, nout, 0)
    else:
        plan.exec_batch_dev(gx.ptr, nx, ldx, ncols, c["n0"], c["acc0"], c["delta"], go.ptr, nout, 0)
    device.sync()
    assert np.array_equal(gx.data(), X.ravel(order="F"))
    y = go.data((nout, ncols))
    # the host form: the same kernel behind a staged copy; NaN cells after the output must survive
    hbuf = np.full(nout * ncols + GUARD, np.nan, dtype=eo)
    if c["entry"] == "exec_dev":
        plan.exec(np.ascontiguousarray(X[:, 0]), nx, c["n0"], c["acc0"], c["delta"], hbuf, nout)
    else:
        plan.exec_batch(np.asfortranarray(X), nx, ldx, ncols, c["n0"], c["acc0"], c["delta"], hbuf, nout)
    assert np.isnan(hbuf[nout * ncols:]).all()
    assert np.array_equal(_bits(hbuf[:nout * ncols].reshape((nout, ncols), order="F")), _bits(y)), "host != device"
    plan.close()
    ph = ExactPhase(c["acc0"], c["delta"], N)
    ratio = check_outputs(y, X[:nx], pfb, dpfb, c["n0"], ph, np.arange(nout), True, f"{dx}-{dh} N={N} {c['entry']}")
    _note(dx, dh, False, ratio)


# =============================================================================== GPU: every instance and regime, exact

@pytest.mark.gpu
@pytest.mark.parametrize("dx,dh", TRIPLES, ids=TRIPLE_IDS)
def test_one_shot_exact(dsp, dx, dh):
    cases = [c for c in one_shot_cases() if c["dx"] == dx and c["dh"] == dh]
    assert cases
    for k, c in enumerate(cases):
        _run_one_shot(dsp, c, 100 + k)


@pytest.mark.gpu
@pytest.mark.parametrize("dx,dh", TRIPLES, ids=TRIPLE_IDS)
def test_stream_exact_with_guarded_histories(dsp, dx, dh):
    """stream_exec_dev chunk by chunk on guarded buffers: inputs between sentinels, outputs (column stride ldo > nout)
    and both history buffers between NaN cells.  Each chunk's outputs against the exact phases of its own call on the
    virtual column [history; chunk], and each new history bit for bit."""
    from dspb200 import device
    for ci, ch in enumerate(c for c in stream_chains() if c["dx"] == dx and c["dh"] == dh):
        rng = np.random.default_rng(200 + ci)
        N, ncols = ch["N"], ch["ncols"]
        h = int_taps(rng, ch["hlen"], dh)
        pfb, dpfb = banks(h, N)
        tpp = pfb.shape[0]
        H = tpp - 1
        plan = dsp._lib.ResampleArbPlan(dx, h, N)
        eo = plan.out_dtype
        calls, delta = _chain_calls(ch)
        hist = np.zeros((H, ncols), dtype=dx)
        gh = [Guarded(dx, H * ncols), Guarded(dx, H * ncols)]
        for k, (nx, deficit, acc0, n0, nout, null) in enumerate(calls):
            x = int_signal(rng, (nx, ncols), dx)
            gx = Guarded(dx, nx * ncols, rng=rng, data=x)
            ldo = nout + 3
            go = Guarded(eo, ldo * ncols)
            hin, hout = gh[k % 2], gh[(k + 1) % 2]
            plan.stream_exec_dev(None if null else hin.ptr, hout.ptr, gx.ptr, nx, ncols, deficit, acc0, delta, go.ptr, ldo,
                                 nout, 0)
            device.sync()
            assert np.array_equal(gx.data(), x.ravel(order="F"))
            if not null:
                assert np.array_equal(hin.data((H, ncols)), hist)      # read, not written
            y = go.data((ldo, ncols))
            assert np.isnan(y[nout:]).all(), "a cell past nout in an output column was written"
            v = np.concatenate([hist, x])
            ratio = check_outputs(y[:nout], v, pfb, dpfb, n0, ExactPhase(acc0, delta, N), np.arange(nout), True,
                                  f"{dx}-{dh} N={N} chunk {k}")
            _note(dx, dh, True, ratio)
            hist = v[v.shape[0] - H:]
            assert np.array_equal(hout.data((H, ncols)), hist), f"new history, chunk {k}"
        plan.close()


@pytest.mark.gpu
def test_large_j_float64(dsp):
    """One Float64 call of 69e6 (~2^26) integer samples at rate 0.98, N = 32: its late outputs have j*delta >= 2^31, where a
    phase formed as acc0 + j*delta in one double is off by ~2^-22 phases, far outside BETA ~ 1.4e-14.  Probes at both
    ends, the middle and around tile edges."""
    from dspb200 import device
    rng = np.random.default_rng(31)
    N, rate, hlen = 32, 0.98, 12 * 32 - 5
    h = int_taps(rng, hlen, F64)
    pfb, dpfb = banks(h, N)
    tpp = pfb.shape[0]
    nx = 69_000_000
    delta, acc0 = N / rate, _undelay_acc(hlen, rate, N)
    n0 = 6
    nout = math.ceil((nx - n0) * rate)
    assert (nout - 1) * delta >= 2 ** 31
    x = rng.integers(-8, 9, nx).astype(np.float64)
    plan = dsp._lib.ResampleArbPlan(F64, h, N)
    dx_ = device.to_device(x)
    dy = device.DeviceArray((nout,), F64)
    plan.exec_dev(dx_.ptr, nx, n0, acc0, delta, dy.ptr, nout, 0)
    device.sync()
    y = dy.to_host()
    plan.close()
    del dx_, dy
    tile = arb_tiling(tpp, N, delta, 8, 8)[0]
    edges = np.arange(tile, nout, tile)
    pick = np.concatenate([edges[:50], edges[len(edges) // 2:len(edges) // 2 + 50], edges[-200:]])
    js = np.unique(np.concatenate([np.arange(0, 2000), np.arange(nout - 4000, nout), np.arange(nout // 2, nout // 2 + 1000),
                                   (pick[:, None] + np.arange(-2, 2)).ravel()]))
    js = js[(js >= 0) & (js < nout)]
    ratio = check_outputs(y[js][:, None], x[:, None], pfb, dpfb, n0, ExactPhase(acc0, delta, N), js, True, "large j")
    _note(F64, F64, False, ratio)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F64, C64, C128], ids=str)
def test_device_firfilter_chunks_exact(dsp, dt):
    """FIRFilter(h, rate, device=True) on 3 channels over chunks of 1, of tpp - 2 and of random lengths: every chunk
    against the exact phases of the (n0, acc0) that _step passes, on the virtual column [history; chunk].  Channel 0
    must equal the host FIRFilter bit for bit."""
    rng = np.random.default_rng(41)
    N, rate = 32, 0.98
    for dh in (F32, F64):
        h = int_taps(rng, 12 * N - 5, dh)
        pfb, dpfb = banks(h, N)
        tpp = pfb.shape[0]
        H = tpp - 1
        fd = dsp.FIRFilter(h, rate, N, device=True)
        fh = dsp.FIRFilter(h, rate, N)
        fd.setphase(fd.timedelay())
        fh.setphase(fh.timedelay())
        hist = np.zeros((H, 3), dtype=dt)
        sizes = [1] * 5 + [tpp - 2] * 4 + [int(v) for v in rng.integers(1, 3000, 12)] + [1, tpp - 2]
        for k, nx in enumerate(sizes):
            x = int_signal(rng, (nx, 3), dt)
            st = fd._step(fd.phi_idx, fd.input_deficit, fd.phi_accumulator, nx)
            y = fd.filt(dsp.to_device(np.asfortranarray(x))).to_host()
            yh = fh.filt(x[:, 0])
            assert y.shape == (st.nout, 3)
            assert np.array_equal(_bits(y[:, 0]), _bits(yh)), f"device != host, chunk {k}"
            v = np.concatenate([hist, x])
            if st.nout:
                eo = y.dtype
                ratio = check_outputs(y, v, pfb, dpfb, st.n0, ExactPhase(st.phase0, fd.delta, N), np.arange(st.nout), True,
                                      f"FIRFilter {dt}/{dh} chunk {k}")
                _note(dt, dh, True, ratio)
                assert eo == out_dtype(dt, dh)
            hist = v[v.shape[0] - H:]


# =============================================================================== GPU: random data, per-output bound

@pytest.mark.gpu
@pytest.mark.parametrize("dx,dh", TRIPLES, ids=TRIPLE_IDS)
def test_random_data_within_bound(dsp, dx, dh):
    """Gaussian samples, resample_filter taps: every output within the per-output rounding bound, one-shot and
    streamed."""
    from dspb200 import device
    rng = np.random.default_rng(51)
    for rate in (0.98, 2.618, 1 / 55.55):
        N = 32
        h = dsp.resample_filter(rate, N).astype(dh)
        pfb, dpfb = banks(h, N)
        tpp = pfb.shape[0]
        delta, acc0 = N / rate, _undelay_acc(h.size, rate, N)
        nout = 2000
        nx = int(nout * delta / N) + 5
        X = rng.standard_normal((nx, 3))
        if _cplx(dx):
            X = X + 1j * rng.standard_normal((nx, 3))
        X = X.astype(dx)
        plan = dsp._lib.ResampleArbPlan(dx, h, N)
        gx = Guarded(dx, nx * 3, rng=rng, data=X)
        go = Guarded(plan.out_dtype, nout * 3)
        plan.exec_batch_dev(gx.ptr, nx, nx, 3, 4, acc0, delta, go.ptr, nout, 0)
        device.sync()
        y = go.data((nout, 3))
        r = check_outputs(y, X, pfb, dpfb, 4, ExactPhase(acc0, delta, N), np.arange(nout), False, f"random {rate}")
        _note(dx, dh, False, r)
        # the same column streamed in three chunks (HIST)
        f = dsp.FIRFilter(h, rate, N, device=True)
        H = tpp - 1
        hist = np.zeros((H, 3), dtype=dx)
        for a, b in ((0, 7), (7, nx // 2), (nx // 2, nx)):
            x = np.asfortranarray(X[a:b])
            st = f._step(f.phi_idx, f.input_deficit, f.phi_accumulator, b - a)
            ys = f.filt(dsp.to_device(x)).to_host()
            v = np.concatenate([hist, x])
            if st.nout:
                r = check_outputs(ys, v, pfb, dpfb, st.n0, ExactPhase(st.phase0, f.delta, N), np.arange(st.nout), False,
                                  f"random streamed {rate}")
                _note(dx, dh, True, r)
            hist = v[v.shape[0] - H:]
        plan.close()


@pytest.mark.gpu
def test_report_largest_ratio():
    """Largest error-to-bound ratio per instance over the tests above (run after them in file order).  The bound of a
    Float32 output is half an ulp plus terms far below it, so its ratio comes close to 1 by construction."""
    for key, ratio in sorted(_RATIOS.items()):
        print(f"largest error / bound, {key}: {ratio:.6f}")
    assert _RATIOS and all(r <= 1.0 for r in _RATIOS.values())
