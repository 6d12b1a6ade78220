"""Every Welch and STFT kernel instance and entry point (csrc/spectral.cu) bin by bin against a float64 reference.

A plan with a power-of-two nfft = N in 256 .. 16384 (Float32) or 256 .. 8192 (Float64) is fused.  Welch runs
`welch_fused_kernel<T, N, CPLX, MODE, G, BATCH>` on one signal or, BATCH, on the columns of a matrix: MODE 0
loads the segments directly, 1 stages them by TMA, 2 also keeps the window in shared memory, 3 in registers; G thread
groups share one CTA.  Which instance runs is chosen on the device from a preference list and the occupancy calculator,
so `dspb200_spec_plan_pin_welch` pins it: every instance runs on the same data, on the same virtual-CTA count, and must
give bit-identical output (the same units land in the same virtual CTA and every mode does the same arithmetic).  STFT
and spectrogram run `stft_fused_kernel<T, N, CPLX, TMA, WIN>` or, for Float32 1024-point aligned calls, the
warp-per-unit `stft_w1k_kernel`; that routing is deterministic and restated below, so that the case table can show what
it reaches.  Any other nfft runs the cuFFT generic path.

The reference forms each segment as the kernels do (`oracle.periodograms.arraysplit(..., f64=False)`: the window product
in Float64, rounded to the signal eltype, src/periodograms.jl:66), widens it to complex128 and transforms it with
np.fft.  The check is per bin, with u the eps of the eltype, E the mean segment energy (by Parseval also the mean bin
power), S_k the reference's mean |X_k|^2 and m the most units one virtual CTA accumulates in registers:

    |P_k - P_ref,k| * r / mult_k  <=  2 c u log2(N) sqrt(S_k E) + (c u log2 N)^2 E + m u S_k,     c = 2

(r = the scale the output was divided by per segment, mult_k = 2 on the interior bins of a one-sided spectrum).  That is
the error of an FFT accurate to c u log2(N) ||x|| per bin, squared, plus the register sum.  Raw STFT columns must hold
|X_k - X_ref,k| <= c u log2(N) ||x_s||, spectrogram columns the Welch bound with m = 1.  A norm over the whole output
would let a tone's bins hide one broken weak bin; per bin nothing hides.  The CPU tests show that a correct
single-precision computation passes the bound and that planted defects fail it.

Inputs sit between sentinel samples of magnitude 10^6, so one read outside the stored range breaks the bound; outputs sit
between NaN cells that must survive every call."""
import math

import numpy as np
import pytest

from oracle import periodograms as op
from oracle import windows as ow

F32, F64, C64, C128 = (np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))
SIZES = (256, 512, 1024, 2048, 4096, 8192, 16384)          # DSP_FUSED_SIZES, spectral.cu
FAMILIES = [(dt, N) for dt in (F32, C64) for N in SIZES] + [(dt, N) for dt in (F64, C128) for N in SIZES if N <= 8192]
H100_SMS = 132
SMEM_OPTIN = 232448        # cudaDevAttrMaxSharedMemoryPerBlockOptin on the H100 (227 KB)
C_FFT = 2.0
GUARD = 64                 # sentinel / NaN cells on each side of a device buffer
SENTINEL = 1e6
VCTAS = 24                 # common virtual-CTA count of the pinned Welch runs (a multiple of 1, 2 and 3 groups)


def _cplx(dt):
    return np.dtype(dt).kind == "c"


def _f64(dt):
    return np.dtype(dt) in (F64, C128)


def _real(dt):
    return F64 if _f64(dt) else F32


def _fam_id(fam):
    dt, N = fam
    return f"{dt.name}-{N}"


def cdiv(a, b):
    return -(-a // b)


# =============================================================================== routing restated from spectral.cu

def fused_size_ok(nfft, f64):
    """fused_size_ok (spectral.cu)."""
    return 256 <= nfft <= (8192 if f64 else 16384) and nfft & (nfft - 1) == 0


def generic_batch(nfft):
    """Segments per cuFFT call of the generic path (generic_prepare)."""
    return min(max((1 << 22) // nfft, 1), 8192)


def host_chunk_segs(itemsize, hop, k):
    """Segments per chunk of the host dspb200_welch_exec: about 32 MiB of new samples, at least 64."""
    return min(max(((32 << 20) // itemsize) // hop, 64), k)


def padded_len(f64, n):
    """padded_len<T>(n) (fft_core.cuh): the padded data buffer, in complex elements."""
    K = 1 if f64 else 2
    if f64:
        p256 = 4 if n == 512 else (2 if n in (1024, 8192) else 1)
        p4096 = 1 if n == 8192 else 0
    else:
        p256 = 8 if n == 512 else (4 if n in (1024, 8192) else 2)
        p4096 = 2 if n == 8192 else (4 if n == 16384 else 0)
    return ((n - 1) + K * ((n - 1) >> 4) + p256 * ((n - 1) >> 8) + p4096 * ((n - 1) >> 12) + 1 + 3) & ~3


def last_radix(n):
    """fft_last_radix (fft_core.cuh): (radix of the last pass, values per row of its table)."""
    ql = int(math.log2(n)) - 4
    nmid = 0 if ql <= 4 else (1 if ql <= 8 else 2)
    rl = 1 << (ql - 4 * nmid)
    return rl, 0 if rl == 16 else (1 if n == 16384 else rl // 2)


def fft_smem_elems(f64, N):
    """fft_smem_elems<T, N> (fft_core.cuh): data buffer + twiddle tables staged in shared memory."""
    row = 8 if N == 16384 else 6
    e = padded_len(f64, N) + (16 * row if N >= 256 else 0) + (256 * row if N >= 4096 else 0)
    if not f64 and N in (512, 1024, 2048, 16384):
        rl, tlk = last_radix(N)
        e += (N // rl) * tlk
    return e


def welch_smem(dt, N, mode, n, hop, g):
    """welch_layout<T, N, CPLX, MODE>::total(n, hop, G): tables, window (MODE 2), then per group data + staging + mbarrier."""
    f64, cplx = _f64(dt), _cplx(dt)
    csz = 16 if f64 else 8
    pl = padded_len(f64, N)
    tables = (fft_smem_elems(f64, N) - pl) * csz
    window = n * 8 if mode == 2 else 0
    stage = (n if cplx else hop + n) if mode >= 1 else 0
    group = ((pl * csz + stage * dt.itemsize + 15) & ~15) + 16
    return tables + window + g * group


def welch_candidates(dt, N, aligned, windowed):
    """The preference list of welch_candidates in csrc/spectral.cu, in order: (MODE, G)."""
    f32, cplx = not _f64(dt), _cplx(dt)
    multi = f32 and 1024 <= N <= 4096
    wreg = f32 and N <= 4096
    c = []
    if aligned:
        if windowed:
            if cplx:
                c += [(3, 1)] if wreg else []
                c += [(2, 1)]
                c += [(3, 2), (2, 2)] if multi else []
            else:
                c += [(2, 3), (2, 2)] if multi else []
                c += [(2, 1)]
                c += [(3, 1)] if wreg else []
        c += [(1, 3)] if multi and not cplx else []
        c += [(1, 1)]
        c += [(1, 2)] if multi else []
    c += [(0, 1)]                                    # offered when nothing above fits
    return c


def welch_instances(dt, N):
    """Every compiled (MODE, G) of one (eltype, N): the union of the preference lists."""
    return sorted({mg for a in (False, True) for w in (False, True) for mg in welch_candidates(dt, N, a, w)})


def welch_aligned(dt, base_aligned, n, hop, length=None, nchan=1):
    """The TMA alignment class of a Welch call (segment starts, hop, n and, batched, the channel stride)."""
    esz = dt.itemsize
    stride_ok = nchan == 1 or length is None or (length * esz) % 16 == 0
    return base_aligned and stride_ok and (hop * esz) % 16 == 0 and (n * esz) % 16 == 0


W1K_TABLE, W1K_DATA, W1K_WARPS = 32 * 16, 1216, 4


def w1k_smem(dt, n, hop, windowed):
    """Dynamic shared memory of stft_w1k_kernel (launch_stft_fused)."""
    stage = n if _cplx(dt) else hop + n
    warp = ((W1K_DATA * 8 + stage * dt.itemsize + 15) & ~15) + 16
    return W1K_TABLE * 8 + (n * 8 if windowed else 0) + W1K_WARPS * warp


def stft_route(dt, N, n, hop, length, nchan, base_aligned, windowed):
    """The kernel launch_stft_fused runs for a one-shot call: ("w1k", dtype, WIN) or ("fused", dtype, N, TMA, WIN).
    (A stream runs the route of an aligned call of its plan; tests/test_stft_stream.py.)"""
    f64, cplx = _f64(dt), _cplx(dt)
    esz = dt.itemsize
    aligned = base_aligned and ((length * esz) % 16 == 0 or nchan == 1) and (hop * esz) % 16 == 0 and (n * esz) % 16 == 0
    w1k = not f64 and N == 1024
    if w1k and aligned:
        assert w1k_smem(dt, n, hop, windowed) <= SMEM_OPTIN
        return ("w1k", dt.name, int(windowed))
    base = fft_smem_elems(f64, N) * (16 if f64 else 8)
    stage = (n if cplx else hop + n) * esz + 16
    tma = not w1k and aligned and base + stage <= SMEM_OPTIN and (base + stage <= 100 * 1024 or N >= 8192)
    return ("fused", dt.name, N, tma, -1 if f64 else int(windowed))


def stft_instances():
    """Every stft_fused_kernel instance that launch_stft_fused can reach, and the four stft_w1k_kernel instances: all the
    STFT instances spectral.cu compiles, which one-shot and streaming calls share."""
    inst = set()
    for dt, N in FAMILIES:
        for tma in (False, True):
            if tma and not _f64(dt) and N == 1024:
                continue                             # aligned Float32 1024-point calls run stft_w1k_kernel
            for win in ((-1,) if _f64(dt) else (0, 1)):
                inst.add(("fused", dt.name, N, tma, win))
    for dt in (F32, C64):
        for win in (0, 1):
            inst.add(("w1k", dt.name, win))
    return inst


def stft_unit_forms(dt, N, n, k):
    """stft_fused_kernel's unit forms: FAST (n == N, complex or both real segments present) and the general one."""
    units = k if _cplx(dt) else cdiv(k, 2)
    forms = set()
    for u in range(units):
        hasB = not _cplx(dt) and 2 * u + 1 < k
        forms.add("fast" if n == N and (_cplx(dt) or hasB) else "general")
    return forms


def stft_emit_forms(dt, N, n, k, onesided, psd_only):
    """stft_emit specialisations (MODE, HASB, ONES, ACC) stft_unit picks per psd_only."""
    cplx = _cplx(dt)
    out = set()
    for form in stft_unit_forms(dt, N, n, k):
        hb = (0 if cplx else 1) if form == "fast" else -1
        if psd_only & 2:
            out.add((1, -1, -1, True))
        elif psd_only:
            out.add((1, hb, 0 if (cplx or not onesided) else 1, False))
        else:
            out.add((0, hb, -1, False))
    return out


# =============================================================================== reference and bound

def window_of(kind, n, rng):
    if kind is None:
        return None
    if kind == "hann":
        return ow.hanning(n)
    if kind == "ones":
        return np.ones(n)
    if kind == "rand":                                   # asymmetric, positive: a reversed read changes every product
        return 0.25 + rng.random(n)
    raise ValueError(kind)


def signal(rng, shape, dt):
    g = rng.standard_normal(shape)
    if _cplx(dt):
        g = g + 1j * rng.standard_normal(shape)
    return g.astype(dt)


def ref_segments(x, n, hop, nfft, window):
    """Segments as the kernels form them (window product rounded to the eltype), their complex128 spectra (k x nfft) and
    energies."""
    segs = op.arraysplit(x, n, n - hop, nfft, window, f64=False)
    wide = segs.astype(np.complex128)
    return np.fft.fft(wide, axis=1), np.sum(np.abs(wide) ** 2, axis=1)


def norm2_of(window, n):
    return float(n) if window is None else float(np.sum(np.abs(window) ** 2))


def bins_and_mult(nfft, onesided):
    if not onesided:
        return np.arange(nfft), np.ones(nfft)
    b = np.arange(nfft // 2 + 1)
    mult = np.full(b.size, 2.0)
    mult[0] = 1.0
    if nfft % 2 == 0:
        mult[-1] = 1.0
    return b, mult


def power_bound(S, E, u, N, m):
    cu = C_FFT * u * math.log2(N)
    return 2 * cu * np.sqrt(S * E) + cu * cu * E + m * u * S


def check_power(P, S, E, mult, scale, u, N, m, what=""):
    """|P * scale / mult - S| within power_bound, bin by bin (NaN fails).  Returns the largest error-to-bound ratio."""
    P = np.asarray(P, dtype=np.float64)
    err = np.abs(P * scale / mult - S)
    bound = power_bound(S, E, u, N, m)
    ok = err <= bound
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, (what, bad[:8], err[bad[:4]], bound[bad[:4]])
    return float(np.max(err / np.maximum(bound, 1e-300))) if err.size else 0.0


def check_welch(P, X, en, nfft, onesided, r, u, m, what=""):
    """A Welch average of the k = X.shape[0] reference segments, computed with r (per segment: r / k)."""
    b, mult = bins_and_mult(nfft, onesided)
    S = np.mean(np.abs(X) ** 2, axis=0)[b]
    return check_power(P, S, float(np.mean(en)), mult, r / X.shape[0], u, nfft, m, what)


def check_stft_raw(Y, X, en, nfft, onesided, u, what=""):
    """Y: nout x k raw columns; X: k x nfft reference spectra; per column |Y - X| <= c u log2(N) ||x_s||."""
    b, _ = bins_and_mult(nfft, onesided)
    err = np.abs(np.asarray(Y, dtype=np.complex128) - X[:, b].T)
    bound = C_FFT * u * math.log2(nfft) * np.sqrt(en)[None, :]
    ok = err <= bound
    assert ok.all(), (what, np.argwhere(~ok)[:8])
    return float(np.max(err / np.maximum(bound, 1e-300))) if err.size else 0.0


def check_stft_psd(Y, X, en, nfft, onesided, r, u, what=""):
    b, mult = bins_and_mult(nfft, onesided)
    worst = 0.0
    for j in range(X.shape[0]):
        worst = max(worst, check_power(Y[:, j], np.abs(X[j, b]) ** 2, float(en[j]), mult, r, u, nfft, 1, (what, j)))
    return worst


def eps(dt):
    return float(np.finfo(_real(dt)).eps)


# =============================================================================== CPU: the bound, the table

def _sp_welch(segs_c64, nfft, onesided, r0, k=None):
    """A correct single-precision Welch of k segments (default: all rows): complex64 FFT (numpy >= 2 transforms it in
    single precision), |X|^2 and the sum over the rows in float32, fft2pow! scaling in Float64."""
    Xs = np.fft.fft(segs_c64, axis=1)
    assert Xs.dtype == C64
    p = (Xs.real * Xs.real + Xs.imag * Xs.imag).astype(F32)
    acc = np.zeros(nfft, F32)
    for row in p:
        acc = (acc + row).astype(F32)
    b, mult = bins_and_mult(nfft, onesided)
    k = segs_c64.shape[0] if k is None else k
    return (acc.astype(np.float64)[b] * mult / (k * r0)).astype(F32), Xs


def _cpu_case(rng, N, cplx, kind, k):
    dt = C64 if cplx else F32
    n, hop = N, N // 2
    x = signal(rng, (k - 1) * hop + n, dt)
    w = window_of(kind, n, rng)
    X, en = ref_segments(x, n, hop, N, w)
    segs = op.arraysplit(x, n, n - hop, N, w, f64=False).astype(C64)
    return x, w, X, en, segs, norm2_of(w, n)


def test_bound_passes_a_correct_single_precision_computation():
    rng = np.random.default_rng(1)
    worst = 0.0
    for N in SIZES:
        for cplx in (False, True):
            for kind in (None, "hann", "rand"):
                for k in (1, 37):
                    _, w, X, en, segs, r0 = _cpu_case(rng, N, cplx, kind, k)
                    onesided = not cplx
                    P, Xs = _sp_welch(segs, N, onesided, r0)
                    worst = max(worst, check_welch(P, X, en, N, onesided, k * r0, eps(F32), k, (N, cplx, kind, k)))
                    b, _ = bins_and_mult(N, onesided)
                    check_stft_raw(Xs[:, b].T, X, en, N, onesided, eps(F32))
                    ps = (np.abs(Xs[:, b]) ** 2).astype(F32).T
                    _, mult = bins_and_mult(N, onesided)
                    check_stft_psd((ps * mult[:, None] / r0).astype(F32), X, en, N, onesided, r0, eps(F32))
    print(f"largest error-to-bound ratio of a single-precision Welch: {worst:.3g}")
    assert worst < 1


def test_bound_rejects_planted_defects():
    rng = np.random.default_rng(2)
    rejected = []
    for N in (256, 4096, 16384):
        k = 37
        x, w, X, en, segs, r0 = _cpu_case(rng, N, False, "rand", k)
        u = eps(F32)
        hop = N // 2

        def welch_fails(bad_segs, name, nyquist_m2=False):
            P, _ = _sp_welch(bad_segs, N, True, r0, k)
            if nyquist_m2:
                P = P.copy()
                P[-1] *= 2
            try:
                check_welch(P, X, en, N, True, k * r0, u, k)
            except AssertionError:
                rejected.append((N, name))
                return
            raise AssertionError(f"{name} passed the bound at N = {N}")

        s = segs.copy()
        s[5, 17] = 0                                                     # one sample dropped from one segment
        welch_fails(s, "dropped sample")
        s = segs.copy()
        s[5, :N] = (x[5 * hop + 1:5 * hop + 1 + N] * w).astype(F32)     # one segment shifted by one sample
        welch_fails(s, "shifted segment")
        s = op.arraysplit(x, N, N - hop, N, w[::-1], f64=False).astype(C64)
        welch_fails(s, "reversed window")
        welch_fails(segs, "Nyquist scaled by m2", nyquist_m2=True)
        welch_fails(segs[:-1], "last segment of odd k dropped")
        welch_fails(np.concatenate([segs, segs[-1:]]), "last segment of odd k duplicated")
        # A and B of one real pair swapped: Welch cannot see it, a spectrogram column must
        b, mult = bins_and_mult(N, True)
        Xs = np.fft.fft(segs, axis=1)
        raw = Xs[:, b].T.copy()
        raw[:, [10, 11]] = raw[:, [11, 10]]
        with pytest.raises(AssertionError):
            check_stft_raw(raw, X, en, N, True, u)
        ps = ((np.abs(raw) ** 2) * mult[:, None] / r0).astype(F32)
        with pytest.raises(AssertionError):
            check_stft_psd(ps, X, en, N, True, r0, u)
        rejected.append((N, "A and B of a real pair swapped"))
        # a neighbouring channel's column
        x2 = signal(rng, x.size, F32)
        X2, _ = ref_segments(x2, N, hop, N, w)
        raw = Xs[:, b].T.copy()
        raw[:, 3] = X2[3, b]
        with pytest.raises(AssertionError):
            check_stft_raw(raw, X, en, N, True, u)
        rejected.append((N, "neighbouring channel's column"))
    for N, name in rejected:
        print(f"rejected at N = {N}: {name}")
    assert len(rejected) == 3 * 8


# ------------------------------------------------------------------------------- case tables

def inst_geometry(dt, N):
    """(n, hop) of the per-instance Welch test: the longest n in N, N/2, ... at which every instance fits, hop = n/2."""
    for n in (N, N // 2, N // 4, N // 8):
        if all(welch_smem(dt, N, m, n, n // 2, g) <= SMEM_OPTIN for m, g in welch_instances(dt, N)):
            return n, n // 2
    raise AssertionError((dt, N))


def inst_segments(dt):
    """k of the per-instance test: 3 VCTAS + 1 units, so every group runs several units and the TMA prefetch chain runs;
    real: an odd k, so the last unit carries one segment."""
    units = 3 * VCTAS + 1
    return units if _cplx(dt) else 2 * units - 1


def welch_shape_cases(dt, N):
    """(n, hop, k, window, onesided) of test_welch_shapes: k in {1, 2, 3, many}; n == N and n < N not a multiple of 16;
    hop 1, aligned, unaligned; staging too large for TMA (hop = n); every window; two-sided real input."""
    cplx = _cplx(dt)
    os_ = not cplx
    cases = [(N, N // 2, k, "hann", os_) for k in (1, 2, 3, 50)]
    cases += [(N - 12, hop, 7, "rand", os_) for hop in (1, 16, 37)]
    cases += [(N, N // 4, 9, kind, os_) for kind in (None, "rand", "ones")]
    cases += [(N, N, 4, "rand", os_)]
    if not cplx:
        cases += [(N, N // 2, 7, "hann", False)]
    return cases


def tma_small_n(dt, N):
    """The longest n in N, N/2, ... whose aligned single-channel STFT stages by TMA (None: the size never does)."""
    n = N
    while n >= 16:
        if stft_route(dt, N, n, n // 2, 0, 1, True, False)[3:4] == (True,) or \
                stft_route(dt, N, n, n // 2, 0, 1, True, False)[0] == "w1k":
            return n
        n //= 2
    return None


def stft_cases(dt, N):
    """(n, hop, k, nchan, len_pad, offset, windowed, onesided) of test_stft_every_instance.  len_pad extra samples per
    channel make the channel stride a multiple of 16 bytes or not."""
    cplx = _cplx(dt)
    os_ = not cplx
    cases = []
    nt = tma_small_n(dt, N)
    for win in (False, True):
        cases.append((N, N // 2, 7, 1, 0, 0, win, os_))
        cases.append((N, N // 2, 7, 1, 0, 1, win, os_))
        if nt is not None and nt != N:
            cases.append((nt, nt // 2, 5, 1, 0, 0, win, os_))
            cases.append((nt, nt // 2, 5, 1, 0, 1, win, os_))
    cases.append((N - 12, 37, 6, 5, 0, 0, True, os_))
    hop = (nt or N) // 4
    n = nt or N
    length = 4 * hop + n
    pad = (-length) % 16
    cases.append((n, hop, 5, 5, pad, 0, False, os_))                # channel stride a multiple of 16 bytes
    cases.append((n, hop, 5, 5, pad + 1, 0, False, os_))            # and not
    if not cplx:
        cases.append((N, N // 2, 5, 1, 0, 0, True, False))
    return cases


def stft_case_len(n, hop, k, len_pad):
    return (k - 1) * hop + n + len_pad


# (dtype, nfft) of the generic-path test: non-powers of two, a size above the fused limit, Float64 16384
GENERIC_CASES = [(F32, 200), (C64, 300), (F32, 1000), (F32, 65536), (F64, 16384)]


def host_chunk_case():
    """(dtype, N, hop) of test_host_welch_exec_odd_chunk: Float32, n = N, 2^25 / 4 / hop odd."""
    N = 4096
    for hop in range(N - 1, N // 2, -1):
        if host_chunk_segs(4, hop, 1 << 30) % 2 == 1:
            return F32, N, hop
    raise AssertionError


def test_restated_routing():
    assert [fused_size_ok(n, False) for n in (128, 256, 1000, 16384, 32768)] == [False, True, False, True, False]
    assert not fused_size_ok(16384, True) and fused_size_ok(8192, True)
    assert [generic_batch(n) for n in (200, 300, 1000, 16384, 65536)] == [8192, 8192, 4194, 256, 64]
    # the warp-per-unit kernel always fits: hop <= n <= 1024, windowed, 4 warps
    assert w1k_smem(F32, 1024, 1024, True) <= 84 * 1024 and w1k_smem(C64, 1024, 1024, True) <= 84 * 1024
    # TMA staging of the STFT: aligned, within the opt-in limit and 100 KB below N = 8192
    assert stft_route(F32, 4096, 4096, 2048, 0, 1, True, True) == ("fused", "float32", 4096, True, 1)
    assert stft_route(F32, 4096, 4096, 2048, 0, 1, False, True) == ("fused", "float32", 4096, False, 1)
    assert stft_route(F32, 1024, 1024, 512, 0, 1, True, False) == ("w1k", "float32", 0)
    assert stft_route(F32, 1024, 1024, 512, 0, 1, False, False) == ("fused", "float32", 1024, False, 0)
    assert stft_route(F32, 4096, 4096, 2048, 4 * 2048 + 4097, 3, True, True)[3] is False     # channel stride
    assert stft_route(F64, 4096, 4096, 2048, 0, 1, True, False)[3] is False                 # above 100 KB
    assert stft_route(F64, 8192, 4096, 2048, 0, 1, True, False)[3] is True                  # N >= 8192: limit only
    assert stft_route(F32, 16384, 16384, 8192, 0, 1, True, False)[3] is False               # above the opt-in limit
    # Welch: the 16384-point Float32 and 8192-point Float64 TMA instances need n well below N to fit
    assert welch_smem(F32, 16384, 1, 16384, 8192, 1) > SMEM_OPTIN and welch_smem(F32, 16384, 1, 4096, 2048, 1) <= SMEM_OPTIN
    assert welch_candidates(F32, 4096, True, True)[:2] == [(2, 3), (2, 2)]
    assert welch_candidates(C64, 4096, True, True)[:2] == [(3, 1), (2, 1)]
    assert welch_candidates(F64, 4096, False, True) == [(0, 1)]
    assert host_chunk_segs(4, 4093, 10 ** 6) == 2049 and host_chunk_segs(8, 1 << 30, 100) == 64


def test_case_table_covers_every_instance():
    # Welch: 109 instances of each kernel, every one runnable at the per-instance geometry
    counts = {}
    for dt, N in FAMILIES:
        inst = welch_instances(dt, N)
        counts[dt.name] = counts.get(dt.name, 0) + len(inst)
        n, hop = inst_geometry(dt, N)
        assert all(welch_smem(dt, N, m, n, hop, g) <= SMEM_OPTIN for m, g in inst)
        assert welch_aligned(dt, True, n, hop) and not welch_aligned(dt, False, n, hop)
        k = inst_segments(dt)
        units = k if _cplx(dt) else cdiv(k, 2)
        assert units > 3 * VCTAS and VCTAS % 6 == 0 and VCTAS <= H100_SMS * 4      # at most the plan's partial rows
        # the shape table: staging too large for every TMA candidate at the largest sizes, hop 1 / aligned / unaligned
        shapes = welch_shape_cases(dt, N)
        assert {k for _, _, k, _, _ in shapes} >= {1, 2, 3, 50}
        assert any(n % 16 and n < N for n, *_ in shapes)
        hops = [(n, hop) for n, hop, *_ in shapes if n < N]
        assert any(h == 1 for _, h in hops) and any(welch_aligned(dt, True, n, h) for n, h in hops)
        assert any(not welch_aligned(dt, True, n, h) for n, h in hops) or dt.itemsize == 16     # ComplexF64: every hop aligned
    print(f"Welch instances per kernel: {counts}, total {sum(counts.values())}")
    assert counts == {"float32": 38, "complex64": 35, "float64": 18, "complex128": 18}
    assert all(welch_smem(dt, N, m, N, N, g) > SMEM_OPTIN for dt, N in ((F32, 16384), (C64, 16384), (F64, 8192), (C128, 8192))
               for m, g in welch_instances(dt, N) if m >= 1)
    # STFT: the case table reaches every reachable instance, the FAST and general unit forms and every emit form
    reach, forms, emits = set(), set(), set()
    for dt, N in FAMILIES:
        for n, hop, k, nchan, pad, off, win, os_ in stft_cases(dt, N):
            length = stft_case_len(n, hop, k, pad)
            route = stft_route(dt, N, n, hop, length, nchan, off == 0, win)
            reach.add(route)
            if route[0] == "fused":
                forms |= {(dt.name, N, f) for f in stft_unit_forms(dt, N, n, k)}
                for psd in (0, 1, 3):
                    emits |= {(_cplx(dt), e) for e in stft_emit_forms(dt, N, n, k, os_, psd)}
    want = stft_instances()
    assert len(want) == 80 - 4 + 4
    assert reach == want, (sorted(want - reach), sorted(reach - want))
    for dt, N in FAMILIES:
        if not (N == 1024 and not _f64(dt)):
            assert {f for d, nn, f in forms if d == dt.name and nn == N} == {"fast", "general"}, (dt, N)
    assert {e for c, e in emits if not c} == {(0, 1, -1, False), (0, -1, -1, False), (1, 1, 1, False), (1, -1, 1, False),
                                              (1, 1, 0, False), (1, -1, 0, False), (1, -1, -1, True)}
    assert {e for c, e in emits if c} == {(0, 0, -1, False), (0, -1, -1, False), (1, 0, 0, False), (1, -1, 0, False),
                                          (1, -1, -1, True)}
    for route in sorted(reach, key=str):
        print("STFT instance reached:", route)
    # the generic path crosses a batch boundary; the host Welch chunk is odd and shorter than k
    for dt, nfft in GENERIC_CASES:
        assert not fused_size_ok(nfft, _f64(dt))
    dt, N, hop = host_chunk_case()
    assert host_chunk_segs(dt.itemsize, hop, 1 << 30) % 2 == 1


# =============================================================================== GPU helpers

@pytest.fixture(scope="module")
def dsp():
    return pytest.importorskip("dspb200")


class Guarded:
    """A device buffer of GUARD cells, `n` data cells (from `offset` cells on) and GUARD cells: sentinels of magnitude
    10^6 (input) or NaN (output) outside the data."""

    def __init__(self, dt, n, rng=None, data=None, offset=0, fill=None):
        from dspb200 import device
        self.dt, self.n, self.lo = np.dtype(dt), n, GUARD + offset
        total = self.lo + n + GUARD
        if rng is None:
            host = np.full(total, np.nan, dtype=dt)
        else:
            s = rng.choice(np.array([-SENTINEL, SENTINEL]), total)
            if _cplx(dt):
                s = s + 1j * rng.choice(np.array([-SENTINEL, SENTINEL]), total)
            host = s.astype(dt)
        if data is not None:
            host[self.lo:self.lo + n] = np.asarray(data).ravel(order="F")
        elif fill is not None:
            host[self.lo:self.lo + n] = fill
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


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype.itemsize in (8, 16) else np.uint32)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _plan(dsp, dt, n, hop, nfft, onesided, window):
    p = dsp._lib.SpecPlan(dt, n, n - hop, nfft, onesided, window)
    assert p.fused == fused_size_ok(nfft, _f64(dt))
    return p


def _welch(dsp, plan, gin, length, r, nout):
    from dspb200 import device
    go = Guarded(_real(plan.dtype), nout)
    plan.welch_dev(gin.ptr, length, r, go.ptr, 0)
    device.sync()
    gin.data()
    return go.data()


def _welch_batch(dsp, plan, gin, length, nchan, r, nout):
    from dspb200 import device
    go = Guarded(_real(plan.dtype), nout * nchan)
    plan.welch_batch_dev(gin.ptr, length, nchan, r, go.ptr, 0)
    device.sync()
    gin.data()
    return go.data((nout, nchan))


def _stft(dsp, plan, gin, length, nchan, r, psd_only, nout, k, prefill=None):
    from dspb200 import device
    odt = _real(plan.dtype) if psd_only else (C128 if _f64(plan.dtype) else C64)
    go = Guarded(odt, nout * k * nchan, data=prefill)
    dsp._lib.check(dsp._lib.lib.dspb200_stft_exec_dev(plan.handle, gin.ptr, length, nchan, float(r), psd_only, go.ptr, None))
    device.sync()
    gin.data()
    return go.data((nout, k * nchan))


_RATIOS = {}


def _note(dt, ratio):
    _RATIOS[_real(dt).name] = max(_RATIOS.get(_real(dt).name, 0.0), ratio)


# =============================================================================== GPU: every Welch instance

@pytest.mark.gpu
@pytest.mark.parametrize("nchan", [0, 3], ids=["single", "batched"])
def test_welch_tma_refill_after_every_read(dsp, nchan):
    # The case that exposed the staging race: 8192-point Float32 segments, 48 KB staged per unit, several units per virtual
    # CTA.  MODE 1 (window read from global memory) used to refill the staging buffer before the barrier that ends the
    # first pass and without a proxy fence, and was off by up to 5 % against MODE 0 / 2 of the same data.
    from dspb200 import device
    rng = np.random.default_rng(11)
    dt, N, n, hop, k = F32, 8192, 8192, 4096, 145
    length = (k - 1) * hop + n
    lb = length + (-length) % 16
    w = window_of("rand", n, rng)
    r = k * norm2_of(w, n)
    cols = max(nchan, 1)
    xb = signal(rng, (lb, cols), dt)
    refs = [ref_segments(xb[:length, c], n, hop, N, w) for c in range(cols)]
    plan = _plan(dsp, dt, n, hop, N, True, w)
    try:
        gb = Guarded(dt, lb * cols, rng, xb)
        out = {}
        for mode in (0, 1, 2):
            plan.pin_welch(nchan > 0, mode, 1, 6)
            P = _welch_batch(dsp, plan, gb, lb, nchan, r, plan.nout) if nchan else \
                _welch(dsp, plan, gb, length, r, plan.nout)[:, None]
            for c in range(cols):
                _note(dt, check_welch(P[:, c], *refs[c], N, True, r, eps(dt), cdiv(k, 2), (mode, c)))
            out[mode] = P
        assert same_bits(out[0], out[1]) and same_bits(out[0], out[2])
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", FAMILIES, ids=[_fam_id(f) for f in FAMILIES])
def test_welch_every_instance(dsp, dt, N):
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 1])
    cplx, u = _cplx(dt), eps(dt)
    n, hop = inst_geometry(dt, N)
    k = inst_segments(dt)
    units = k if cplx else cdiv(k, 2)
    length = (k - 1) * hop + n
    w = window_of("rand", n, rng)
    r = k * norm2_of(w, n)
    onesided = not cplx
    plan = _plan(dsp, dt, n, hop, N, onesided, w)
    x = signal(rng, length, dt)
    X, en = ref_segments(x, n, hop, N, w)
    gin = Guarded(dt, length, rng, x)
    gin1 = Guarded(dt, length, rng, x, offset=1)
    try:
        inst = welch_instances(dt, N)
        first = None
        for mode, g in inst:
            plan.pin_welch(0, mode, g, VCTAS)
            P = _welch(dsp, plan, gin, length, r, plan.nout)
            assert plan.welch_config(0, True) == (mode, g, VCTAS)
            if first is None:
                first = P
                ratio = check_welch(P, X, en, N, onesided, r, u, cdiv(units, VCTAS), "pinned")
                _note(dt, ratio)
            assert same_bits(P, first), (mode, g)
        P = _welch(dsp, plan, gin1, length, r, plan.nout)                   # unaligned: MODE 0, G 1, same virtual CTAs
        if dt.itemsize < 16:                                                # (ComplexF64 elements keep 16-byte alignment)
            assert plan.welch_config(0, False) == (0, 1, VCTAS)
        assert same_bits(P, first)
        # the default choice equals the pinned run of the configuration it reports
        plan.pin_welch(0, -1, 0, 0)
        assert plan.welch_config(0, True) == (-1, 0, 0)
        Pd = _welch(dsp, plan, gin, length, r, plan.nout)
        md, gd, vd = plan.welch_config(0, True)
        assert (md, gd) in inst and vd > 0
        plan.pin_welch(0, md, gd, vd)
        assert same_bits(_welch(dsp, plan, gin, length, r, plan.nout), Pd)
        _note(dt, check_welch(Pd, X, en, N, onesided, r, u, units, "default"))
        # batched: three channels, channel stride a multiple of 16 bytes
        nchan = 3
        lb = length + (-length) % 16
        xb = signal(rng, (lb, nchan), dt)
        refs = [ref_segments(xb[:, c], n, hop, N, w) for c in range(nchan)]
        gb = Guarded(dt, lb * nchan, rng, xb)
        gb1 = Guarded(dt, lb * nchan, rng, xb, offset=1)
        firstb = None
        for mode, g in inst:
            plan.pin_welch(1, mode, g, VCTAS)
            Pb = _welch_batch(dsp, plan, gb, lb, nchan, r, plan.nout)
            assert plan.welch_config(1, True)[:2] == (mode, g)
            if firstb is None:
                firstb = Pb
                for c in range(nchan):
                    _note(dt, check_welch(Pb[:, c], *refs[c], N, onesided, r, u, units, ("batched", c)))
            assert same_bits(Pb, firstb), ("batched", mode, g)
        assert same_bits(_welch_batch(dsp, plan, gb1, lb, nchan, r, plan.nout), firstb)
        if dt.itemsize < 16:
            assert plan.welch_config(1, False)[:2] == (0, 1)
        plan.pin_welch(1, -1, 0, 0)
        Pbd = _welch_batch(dsp, plan, gb, lb, nchan, r, plan.nout)
        mb, gbd, _ = plan.welch_config(1, True)
        for c in range(nchan):
            _note(dt, check_welch(Pbd[:, c], *refs[c], N, onesided, r, u, units, ("batched default", c)))
        print(f"selector {_fam_id((dt, N))} n={n} hop={hop} windowed: single MODE {md} G {gd} ({vd} virtual CTAs), "
              f"batched MODE {mb} G {gbd}")
        # an instance whose staging does not fit is refused, as restated
        big = _plan(dsp, dt, N, N // 2, N, onesided, window_of("rand", N, rng))
        try:
            for mode, g in inst:
                fits = welch_smem(dt, N, mode, N, N // 2, g) <= SMEM_OPTIN
                if fits:
                    big.pin_welch(0, mode, g, VCTAS)
                else:
                    with pytest.raises(dsp._lib.DSPB200Error) as e:
                        big.pin_welch(0, mode, g, VCTAS)
                    assert e.value.code == dsp._lib.EUNSUPPORTED
        finally:
            big.close()
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
def test_welch_pin_refusals(dsp):
    plan = _plan(dsp, F32, 4096, 2048, 4096, True, None)
    try:
        for args, code in (((0, 2, 1, 24), "EUNSUPPORTED"),        # MODE 2 / 3 without a window
                           ((0, 3, 1, 24), "EUNSUPPORTED"),
                           ((0, 0, 2, 24), "EUNSUPPORTED"),        # no such instance
                           ((0, 1, 4, 24), "EUNSUPPORTED"),
                           ((0, 1, 3, 25), "EINVALID"),            # not a multiple of the groups
                           ((0, 1, 1, -3), "EINVALID"),
                           ((0, 1, 1, 1 << 20), "EINVALID")):      # more virtual CTAs than partial rows
            with pytest.raises(dsp._lib.DSPB200Error) as e:
                plan.pin_welch(*args)
            assert e.value.code == getattr(dsp._lib, code), args
        plan.pin_welch(1, 1, 3, 3 << 20)                           # the batched form has no row limit
    finally:
        plan.close()
    gen = _plan(dsp, F32, 1000, 500, 1000, True, None)
    try:
        with pytest.raises(dsp._lib.DSPB200Error) as e:
            gen.pin_welch(0, 0, 1, 0)
        assert e.value.code == dsp._lib.EUNSUPPORTED
    finally:
        gen.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", FAMILIES, ids=[_fam_id(f) for f in FAMILIES])
def test_welch_shapes(dsp, dt, N):
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 2])
    u = eps(dt)
    try:
        for n, hop, k, kind, onesided in welch_shape_cases(dt, N):
            length = (k - 1) * hop + n
            w = window_of(kind, n, rng)
            r = k * norm2_of(w, n)
            x = signal(rng, length, dt)
            X, en = ref_segments(x, n, hop, N, w)
            gin = Guarded(dt, length, rng, x)
            plan = _plan(dsp, dt, n, hop, N, onesided, w)
            try:
                P = _welch(dsp, plan, gin, length, r, plan.nout)
                units = k if _cplx(dt) else cdiv(k, 2)
                _note(dt, check_welch(P, X, en, N, onesided, r, u, units, (n, hop, k, kind, onesided)))
                mode, g, _ = plan.welch_config(0, welch_aligned(dt, True, n, hop))
                fit = [mg for mg in welch_candidates(dt, N, welch_aligned(dt, True, n, hop), w is not None)
                       if welch_smem(dt, N, mg[0], n, hop, mg[1]) <= SMEM_OPTIN]
                assert (mode, g) in fit, ((n, hop, kind), (mode, g), fit)
                if kind == "ones":                                  # win_mul(x, (1, 0)) is exact
                    plain = _plan(dsp, dt, n, hop, N, onesided, None)
                    try:
                        assert same_bits(_welch(dsp, plain, gin, length, k * n, plain.nout), P)
                    finally:
                        plain.close()
            finally:
                plan.close()
    finally:
        device.empty_cache()


# =============================================================================== GPU: every STFT instance

@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", FAMILIES, ids=[_fam_id(f) for f in FAMILIES])
def test_stft_every_instance(dsp, dt, N):
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 3])
    u = eps(dt)
    runs = {}
    try:
        for case in stft_cases(dt, N):
            n, hop, k, nchan, pad, off, win, onesided = case
            length = stft_case_len(n, hop, k, pad)
            xr = np.random.default_rng([N, dt.num, n, hop, k, nchan, pad, int(win), int(onesided)])   # same data per offset
            w = window_of("rand", n, xr) if win else None
            r = norm2_of(w, n)
            x = signal(xr, (length, nchan), dt)
            refs = [ref_segments(x[:, c], n, hop, N, w) for c in range(nchan)]
            X = np.concatenate([a for a, _ in refs])
            en = np.concatenate([b for _, b in refs])
            gin = Guarded(dt, length * nchan, rng, x, offset=off)
            plan = _plan(dsp, dt, n, hop, N, onesided, w)
            try:
                nout = plan.nout
                raw = _stft(dsp, plan, gin, length, nchan, r, 0, nout, k)
                _note(dt, check_stft_raw(raw, X, en, N, onesided, u, case))
                psd = _stft(dsp, plan, gin, length, nchan, r, 1, nout, k)
                _note(dt, check_stft_psd(psd, X, en, N, onesided, r, u, case))
                pre = (rng.random((nout, k * nchan)) * 4).astype(_real(dt))
                acc = _stft(dsp, plan, gin, length, nchan, r, 3, nout, k, prefill=pre)
                assert same_bits(acc, (pre + psd).astype(_real(dt))), case
                route = stft_route(dt, N, n, hop, length, nchan, off == 0, win)
                key = (n, hop, k, nchan, pad, win, onesided)
                if route[0] == "fused" and key in runs:             # the same data through TMA and direct loads
                    assert same_bits(raw, runs[key][0]) and same_bits(psd, runs[key][1]), case
                if route[0] == "fused":
                    runs[key] = (raw, psd)
            finally:
                plan.close()
    finally:
        device.empty_cache()


# =============================================================================== GPU: streaming and the other entry points

@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", [(F32, 4096), (C64, 2048), (F64, 1024), (C128, 512), (F32, 16384)],
                         ids=lambda v: getattr(v, "name", str(v)))
def test_welch_streaming_alternating_alignment(dsp, dt, N):
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 4])
    n, hop = N, N // 2
    k = 41
    length = (k - 1) * hop + n
    w = window_of("hann", n, rng)
    r = k * norm2_of(w, n)
    onesided = not _cplx(dt)
    x = signal(rng, length, dt)
    X, en = ref_segments(x, n, hop, N, w)
    chunks = [(0, 7), (7, 8), (8, 21), (21, 22), (22, 41)]      # 1-segment chunks: fewer units than virtual CTAs
    plan = _plan(dsp, dt, n, hop, N, onesided, w)
    try:
        one = _welch(dsp, plan, Guarded(dt, length, rng, x), length, r, plan.nout)
        for first_off in (0, 1):
            plan.welch_begin_dev(0)
            keep = []
            for i, (b, e) in enumerate(chunks):
                lo, hi = b * hop, (e - 1) * hop + n
                g = Guarded(dt, hi - lo, rng, x[lo:hi], offset=(first_off + i) % 2)
                plan.welch_accumulate_dev(g.ptr, hi - lo, lo, b, e, 0)
                keep.append(g)
            go = Guarded(_real(dt), plan.nout)
            plan.welch_finalize_dev(r, go.ptr, 0)
            device.sync()
            for g in keep:
                g.data()
            P = go.data()
            m = max(e - b for b, e in chunks)
            _note(dt, check_welch(P, X, en, N, onesided, r, eps(dt), m, ("stream", first_off)))
            _note(dt, check_welch(one, X, en, N, onesided, r, eps(dt), k, "one call"))
            assert plan.welch_config(0, True)[1] > 0
            assert plan.welch_config(0, False)[1] > 0 or dt.itemsize == 16       # ComplexF64: every chunk aligned
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
def test_host_welch_exec_odd_chunk(dsp):
    dt, N, hop = host_chunk_case()
    rng = np.random.default_rng(5)
    chunk = host_chunk_segs(dt.itemsize, hop, 1 << 30)
    k = chunk + 9
    length = (k - 1) * hop + N
    w = window_of("hann", N, rng)
    r = k * norm2_of(w, N)
    x = signal(rng, length, dt)
    plan = _plan(dsp, dt, N, hop, N, True, w)
    try:
        out = np.full(plan.nout, np.nan, dtype=F32)
        plan.welch(x, r, out)
        X, en = ref_segments(x, N, hop, N, w)
        _note(dt, check_welch(out, X, en, N, True, r, eps(dt), cdiv(chunk, 2), ("host", chunk)))
    finally:
        plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", [(F32, 1024), (C64, 4096), (F64, 2048), (F32, 1000)], ids=lambda v: getattr(v, "name", str(v)))
def test_host_stft_equals_device_stft(dsp, dt, N):
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 6])
    n, hop, k, nchan = N, N // 4, 9, 3
    length = (k - 1) * hop + n + 3
    w = window_of("rand", n, rng)
    x = np.asfortranarray(signal(rng, (length, nchan), dt))
    plan = _plan(dsp, dt, n, hop, N, not _cplx(dt), w)
    try:
        for psd in (0, 1):
            odt = _real(dt) if psd else (C128 if _f64(dt) else C64)
            host = np.full((plan.nout, k * nchan), np.nan, dtype=odt, order="F")
            plan.stft(x, length, nchan, norm2_of(w, n), psd, host)
            dev = _stft(dsp, plan, Guarded(dt, length * nchan, rng, x), length, nchan, norm2_of(w, n), psd, plan.nout, k)
            assert same_bits(np.asfortranarray(host), np.asfortranarray(dev)), psd
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,nfft", GENERIC_CASES, ids=[f"{d.name}-{n}" for d, n in GENERIC_CASES])
def test_generic_path_across_batches(dsp, dt, nfft):
    from dspb200 import device
    rng = np.random.default_rng([nfft, dt.num, 7])
    n, hop = nfft, nfft
    k = generic_batch(nfft) + 3
    length = (k - 1) * hop + n
    w = window_of("rand", n, rng)
    r0 = norm2_of(w, n)
    onesided = not _cplx(dt)
    x = signal(rng, length, dt)
    X, en = ref_segments(x, n, hop, nfft, w)
    gin = Guarded(dt, length, rng, x)
    plan = _plan(dsp, dt, n, hop, nfft, onesided, w)
    assert not plan.fused
    try:
        P = _welch(dsp, plan, gin, length, k * r0, plan.nout)
        _note(dt, check_welch(P, X, en, nfft, onesided, k * r0, eps(dt), 1, "generic welch"))
        raw = _stft(dsp, plan, gin, length, 1, r0, 0, plan.nout, k)
        _note(dt, check_stft_raw(raw, X, en, nfft, onesided, eps(dt), "generic stft"))
        psd = _stft(dsp, plan, gin, length, 1, r0, 1, plan.nout, k)
        _note(dt, check_stft_psd(psd, X, en, nfft, onesided, r0, eps(dt), "generic spectrogram"))
    finally:
        plan.close()
        device.empty_cache()


# =============================================================================== GPU: multitaper

def _tapers(n, nt):
    t = ow.dpss(n, 4, nt)
    t = np.asarray(t, dtype=np.float64)
    t = t.T if t.shape[0] == n else t
    return t / np.sqrt(np.sum(t * t, axis=1, keepdims=True))          # r_t = sum w^2: unit power per taper


@pytest.mark.gpu
@pytest.mark.parametrize("dt,nfft", [(F32, 1024), (F32, 2048), (C64, 4096), (F64, 512), (F32, 1000)],
                         ids=lambda v: getattr(v, "name", str(v)))
def test_mt_spectrogram_is_the_float_sum_of_taper_spectrograms(dsp, dt, nfft):
    from dspb200 import device
    rng = np.random.default_rng([nfft, dt.num, 8])
    n, hop, k, nt = nfft, nfft // 2, 6, 4
    length = (k - 1) * hop + n
    onesided = not _cplx(dt)
    tapers = _tapers(n, nt)
    x = signal(rng, length, dt)
    mt = dsp._lib.MtPlan(dt, n, n - hop, nfft, onesided, tapers)
    try:
        gin = Guarded(dt, length, rng, x)
        go = Guarded(_real(dt), mt.nout * k)
        mt.mt_spectrogram_dev(gin.ptr, length, go.ptr, 0)
        device.sync()
        got = go.data((mt.nout, k))
        acc = None
        for t in range(nt):
            p = _plan(dsp, dt, n, hop, nfft, onesided, tapers[t])
            try:
                col = _stft(dsp, p, gin, length, 1, 1.0, 1, p.nout, k)
            finally:
                p.close()
            acc = col if acc is None else (acc + col).astype(_real(dt))
        assert same_bits(got, acc)
    finally:
        mt.close()
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", [(F32, 2048), (F32, 4096), (C64, 1024)], ids=lambda v: getattr(v, "name", str(v)))
def test_mt_pgram_pinned_groups(dsp, dt, N):
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 9])
    nt = 5
    tapers = _tapers(N, nt)
    onesided = not _cplx(dt)
    x = signal(rng, N, dt)
    mt = dsp._lib.MtPlan(dt, N, 0, N, onesided, tapers)
    try:
        Xs, ens = [], []
        for t in range(nt):
            X, en = ref_segments(x, N, N, N, tapers[t])
            Xs.append(X)
            ens.append(en)
        X, en = np.concatenate(Xs), np.concatenate(ens)
        gin = Guarded(dt, N, rng, x)
        res = []
        fit = [mg for mg in welch_instances(dt, N) if welch_smem(dt, N, mg[0], N, N, mg[1]) <= SMEM_OPTIN]
        assert max(g for _, g in fit) >= 2
        for mode, g in (max(fit, key=lambda mg: (mg[1], mg[0])), (1, 1), (0, 1)):
            mt.pin_welch(0, mode, g, 6)
            go = Guarded(_real(dt), mt.nout)
            mt.mt_pgram_dev(gin.ptr, N, go.ptr, 0)
            device.sync()
            gin.data()
            P = go.data()
            _note(dt, check_welch(P, X, en, N, onesided, 1.0, eps(dt), nt, ("mt_pgram", mode, g)))
            res.append(P)
        assert all(same_bits(P, res[0]) for P in res)
    finally:
        mt.close()
        device.empty_cache()


# =============================================================================== GPU: zeros

@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", [(F32, 2048), (C64, 4096), (F64, 8192), (F32, 1024), (F32, 1000)],
                         ids=lambda v: getattr(v, "name", str(v)))
def test_all_zero_signal_gives_positive_zero(dsp, dt, N):
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 10])
    n, hop, k = N, N // 2, 3
    length = (k - 1) * hop + n
    w = window_of("hann", n, rng)
    plan = _plan(dsp, dt, n, hop, N, not _cplx(dt), w)
    try:
        z = np.zeros(length, dtype=dt)
        gin = Guarded(dt, length, rng, z)
        outs = []
        if plan.fused:
            inst = welch_instances(dt, N)
            mode, g = max(inst, key=lambda mg: mg[1])
            plan.pin_welch(0, mode, g, 4 * g)                        # more virtual CTAs than units: idle groups
        outs.append(_welch(dsp, plan, gin, length, k * 1.0, plan.nout))
        gb = Guarded(dt, length * 2, rng, np.zeros(length * 2, dtype=dt))
        outs.append(_welch_batch(dsp, plan, gb, length, 2, k * 1.0, plan.nout))
        for psd in (0, 1):
            outs.append(_stft(dsp, plan, gin, length, 1, 1.0, psd, plan.nout, k))
        for o in outs:
            assert not _bits(o).any(), "not +0"
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
def test_report_largest_ratio():
    # runs last in this module: the largest error-to-bound ratio seen per eltype
    for name, ratio in sorted(_RATIOS.items()):
        print(f"largest error-to-bound ratio {name}: {ratio:.3g}")
        assert ratio <= 1.0
