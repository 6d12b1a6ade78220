"""Oracle: filt / conv core (reference src/dspbase.jl). TEST INFRASTRUCTURE ONLY.

1-D (column-batched) restatement; N-D overlap-save, IIR and deconv are outside
the hot-path scope (SURVEY.md section 8).
"""
import math
import numpy as np
import scipy.fft as sfft

from .util import nextfastfft

SMALL_FILT_CUTOFF = 66  # src/dspbase.jl:3
FFT_TYPES = (np.float32, np.float64, np.complex64, np.complex128)  # src/dspbase.jl:674


def promote(*dts):
    return np.result_type(*dts)


# --------------------------------------------------------------------------- filt (FIR)

def fma_f32(a, b, c):
    """Exact Float32 fused multiply-add, vectorised: round_f32(a*b + c) with ONE rounding.
    a*b is exact in Float64; the Float64 sum is corrected to round-to-odd whenever it is inexact and sits on a
    Float32 rounding boundary, so the final cast cannot double-round."""
    a = np.asarray(a, dtype=np.float32).astype(np.float64)
    b = np.asarray(b, dtype=np.float32).astype(np.float64)
    c = np.asarray(c, dtype=np.float32).astype(np.float64)
    p = a * b
    s = p + c
    bb = s - p                                  # TwoSum error term: s + e == p + c exactly
    e = (p - (s - bb)) + (c - bb)
    bits = s.view(np.int64)
    tie = ((bits & 0x1FFFFFFF) == 0x10000000) & (e != 0) & np.isfinite(s)
    if np.any(tie):
        s = s.copy()
        up = tie & (e > 0)
        dn = tie & (e < 0)
        s[up] = np.nextafter(s[up], np.inf)
        s[dn] = np.nextafter(s[dn], -np.inf)
    return s.astype(np.float32)


def _two_sum(a, b):
    """s = a + b rounded, and the exact error e: s + e == a + b (Knuth's TwoSum, any order of magnitude)."""
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    """Veltkamp split: a == hi + lo exactly, hi and lo with at most 26 significant bits each."""
    t = a * 134217729.0                         # 2^27 + 1
    hi = t - (t - a)
    return hi, a - hi


def fma_f64(a, b, c):
    """Exact Float64 fused multiply-add, vectorised: round_f64(a*b + c) with ONE rounding (Boldo & Melquiond, "Emulation
    of FMA and correctly rounded sums: proved algorithms using rounding to odd", IEEE TC 2008).  a*b = uh + ul exactly
    (Dekker's TwoProduct over a Veltkamp split); c + uh = th + tl exactly (TwoSum); v = tl + ul rounded to odd (the
    rounded sum, moved one ulp towards the TwoSum error when it is inexact and even); result th + v rounded once.
    Valid domain: finite a, b, c whose magnitudes, and that of a*b, are zero or within [2^-900, 2^900] -- so no split,
    product or sum overflows and every low part is a normal number (no subnormal results)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    c = np.asarray(c, dtype=np.float64)
    uh = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    ul = ((ah * bh - uh) + ah * bl + al * bh) + al * bl
    th, tl = _two_sum(c, uh)
    v, e = _two_sum(tl, ul)
    odd = (v.view(np.int64) & 1) == 1
    fix = (e != 0) & ~odd
    if np.any(fix):
        v = np.where(fix, np.nextafter(v, np.where(e > 0, np.inf, -np.inf)), v)
    return th + v


def cmuladd(z, w, x):
    """Base.muladd(z::Complex, w::Complex, x::Complex) (base/complex.jl), vectorised, for complex64 / complex128:
    Complex(muladd(zr, wr, -muladd(zi, wi, -xr)), muladd(zr, wi, muladd(zi, wr, xi))), each muladd an exact fma."""
    z, w, x = np.asarray(z), np.asarray(w), np.asarray(x)
    T = np.result_type(z, w, x)
    f = fma_f32 if T == np.complex64 else fma_f64
    re = f(z.real, w.real, -f(z.imag, w.imag, -x.real))
    im = f(z.real, w.imag, f(z.imag, w.real, x.imag))
    out = np.empty(np.broadcast(z, w, x).shape, dtype=T)
    out.real, out.imag = re, im
    return out


def muladd(a, b, c, T):
    """muladd(a, b, c) in eltype T as Julia evaluates it on FMA hardware: one exact fma for Float32 / Float64, Base.muladd
    for Complex, plain a*b + c otherwise (integers: exact)."""
    T = np.dtype(T)
    if T == np.float32:
        return fma_f32(a, b, c)
    if T == np.float64:
        return fma_f64(a, b, c)
    if T in (np.complex64, np.complex128):
        return cmuladd(np.asarray(a, dtype=T), np.asarray(b, dtype=T), np.asarray(c, dtype=T))
    return (np.asarray(a, dtype=T) * np.asarray(b, dtype=T) + np.asarray(c, dtype=T)).astype(T)


def filt_fir_literal(b, x):
    """Literal transposed direct-form-II loop, src/dspbase.jl:95-105 (one column).

    Pure-Python: small cases only.  Arithmetic in promote_type(eltype(b), eltype(x));
    `muladd` is evaluated as a fused multiply-add (what LLVM emits on FMA hardware),
    emulated by forming the product/sum in the next wider precision.
    """
    b = np.asarray(b)
    x = np.asarray(x)
    T = promote(b.dtype, x.dtype)
    wide = np.complex128 if np.issubdtype(T, np.complexfloating) else np.float64
    if T in (np.float64, np.complex128):
        wide = np.clongdouble if np.issubdtype(T, np.complexfloating) else np.longdouble
    nb = len(b)
    out = np.zeros(len(x), dtype=T)
    si = np.zeros(max(nb - 1, 1), dtype=T)
    bw = b.astype(wide)
    silen = nb - 1

    def fma(a, c, d):
        if T == np.float32:
            return fma_f32(a, c, d)[()]
        return np.asarray(wide(a) * wide(c) + wide(d)).astype(T)[()]

    for i in range(len(x)):
        xi = x[i]
        if silen == 0:
            out[i] = np.asarray(wide(xi) * bw[0]).astype(T)[()]
            continue
        out[i] = fma(xi, b[0], si[0])
        for j in range(silen - 1):
            si[j] = fma(xi, b[j + 1], si[j + 1])
        si[silen - 1] = np.asarray(wide(b[silen]) * wide(xi)).astype(T)[()]
    return out


def filt(b, a, x, f64=False):
    """filt(b, a, x) for length(a)==1, src/dspbase.jl:14-15, 26-66, 95-105.

    y[i] = sum_k (b[k]/a[1]) x[i-k+1] along dim 0 for every column; result eltype
    promote_type(eltype(b), eltype(a), eltype(x)).  Evaluated with the reference's
    accumulation order (oldest tap first, one fused multiply-add per tap) in the
    result dtype, or in double precision when f64=True.
    """
    b = np.atleast_1d(np.asarray(b))
    a = np.atleast_1d(np.asarray(a))
    x = np.asarray(x)
    if b.size == 0:
        raise ValueError("filter vector b must be non-empty")  # ArgumentError :28
    if a.size == 0:
        raise ValueError("filter vector a must be non-empty")  # :29
    if a[0] == 0:
        raise ValueError("filter vector a[1] must be nonzero")  # :30
    if a.size != 1:
        raise NotImplementedError("IIR filt is outside the hot-path scope")
    T = promote(b.dtype, a.dtype, x.dtype)
    if not np.issubdtype(T, np.inexact):
        T = np.dtype(np.float64)
    if x.shape[0] == 0:
        return np.zeros(x.shape, dtype=T)
    if a[0] != 1:
        b = (b / a[0])  # :43-47
    W = (np.complex128 if np.issubdtype(T, np.complexfloating) else np.float64)
    Tout = W if f64 else T
    bT = b.astype(Tout)
    nb = len(bT)
    x2 = x.reshape(x.shape[0], -1).astype(Tout)
    nx = x2.shape[0]
    if nb == 1:  # :40 simple scaling
        return (x2 * bT[0]).astype(Tout).reshape(x.shape)
    xp = np.concatenate([np.zeros((nb - 1, x2.shape[1]), dtype=Tout), x2], axis=0)
    # oldest tap first: acc = b[nb]*x[i-nb+1]; acc = fma(x[i-j+1], b[j], acc) for j = nb-1..1
    acc = (xp[0:nx].astype(W) * W(bT[nb - 1])).astype(Tout)
    exact32 = np.dtype(Tout) == np.float32
    for j in range(nb - 2, -1, -1):
        seg = xp[nb - 1 - j: nb - 1 - j + nx]
        if exact32:
            acc = fma_f32(seg, bT[j], acc)
        else:
            acc = (seg.astype(W) * W(bT[j]) + acc.astype(W)).astype(Tout)
    return acc.reshape(x.shape)


# --------------------------------------------------------------------------- overlap-save planning

def os_fft_complexity(nfft, nb):
    """src/dspbase.jl:262."""
    return (nfft * math.log2(nfft) + nfft) / (nfft - nb + 1)


def optimalfftfiltlength(nb, nx):
    """src/dspbase.jl:268-291."""
    nfull = nb + nx - 1
    first_pow2 = math.ceil(math.log2(nb))
    max_pow2 = math.ceil(math.log2(nfull))
    prev = os_fft_complexity(2 ** first_pow2, nb)
    pow2 = first_pow2 + 1
    while pow2 <= max_pow2:
        new = os_fft_complexity(2 ** pow2, nb)
        if new > prev:
            break
        prev = new
        pow2 += 1
    nfft = 2 ** max_pow2 if pow2 > max_pow2 else 2 ** (pow2 - 1)
    if nfft > nfull:
        nfft = nextfastfft(nfull)
    return nfft


# --------------------------------------------------------------------------- conv kernels (1-D)

def _fft_dt(T):
    return np.dtype(T)


def conv_kern_os(u, v, nfft, nout=None, f64=False, batched=False):
    """1-D restatement of unsafe_conv_kern_os!, src/dspbase.jl:490-609 (+ edge blocks :371-486,
    buffers/plans :299-318, block transform :337-356).  Requires len(u) >= len(v).
    Output eltype promote_type; arithmetic (incl. FFT) in that precision unless f64.
    """
    u = np.asarray(u)
    v = np.asarray(v)
    T = promote(u.dtype, v.dtype)
    if f64:
        T = np.dtype(np.complex128 if np.issubdtype(T, np.complexfloating) else np.float64)
    cplx = np.issubdtype(T, np.complexfloating)
    su, sv = len(u), len(v)
    sout = su + sv - 1 if nout is None else nout
    out = np.zeros(sout, dtype=T)
    ideal_save = nfft - sv + 1
    sout_deficit = max(0, ideal_save - sout)  # :502-504
    save = ideal_save - sout_deficit           # :506
    nblocks = -(-sout // save)                  # cld :507
    uT = u.astype(T)
    # filter transform, scaled once by 1/nfft (:514-516)
    td = np.zeros(nfft, dtype=T)
    td[:sv] = v.astype(T)
    if cplx:
        filter_fd = sfft.fft(td)
    else:
        filter_fd = sfft.rfft(td)
    filter_fd = (filter_fd * (1.0 / nfft)).astype(filter_fd.dtype)

    def block(tdbuff):
        if cplx:  # :348-356, one in-place buffer, unnormalised inverse
            return sfft.ifft(sfft.fft(tdbuff) * filter_fd, norm="forward").astype(T)
        return sfft.irfft(sfft.rfft(tdbuff) * filter_fd, n=nfft, norm="forward").astype(T)  # brfft :337-345

    first_center = -(-(sv - 1) // save) + 1   # cld(sv-1, save)+1  :519
    last_center = su // save                   # fld :520
    if last_center > 1:                         # :527-529
        edge_blocks = list(range(1, first_center)) + list(range(last_center + 1, nblocks + 1))
        center_blocks = range(first_center, last_center + 1)
    else:
        edge_blocks = list(range(1, nblocks + 1))
        center_blocks = range(0)
    for bi in edge_blocks:                      # :371-486 (1-D)
        data_offset = save * (bi - 1)
        pad_before = max(0, sv - data_offset - 1)
        data_ideal_stop = data_offset + save
        pad_after = max(0, data_ideal_stop - su)
        lo = data_offset - sv + pad_before + 1   # 0-based start in u
        hi = data_ideal_stop - pad_after          # exclusive
        tdbuff = np.zeros(nfft, dtype=T)
        if hi > lo:
            tdbuff[pad_before: pad_before + (hi - lo)] = uT[lo:hi]
        y = block(tdbuff)
        block_out_stop = min(data_offset + save, sout)
        u_deficit = max(0, pad_after - sv + 1)
        valid = y[sv - 1: nfft - u_deficit - sout_deficit]
        n = block_out_stop - data_offset
        out[data_offset: data_offset + n] = valid[:n]
    if batched and len(center_blocks) > 0:      # same arithmetic, many blocks per pocketfft call (multi-threaded)
        b_lo, b_hi = center_blocks[0], center_blocks[-1]
        start = save * (b_lo - 1) - sv + 1
        nrows = b_hi - b_lo + 1
        rows = np.lib.stride_tricks.as_strided(uT[start:], shape=(nrows, nfft),
                                               strides=(save * uT.itemsize, uT.itemsize), writeable=False)
        slab = max(1, (1 << 23) // nfft)
        for r0 in range(0, nrows, slab):
            blk = rows[r0: r0 + slab]
            if cplx:
                yb = sfft.ifft(sfft.fft(blk, axis=1) * filter_fd[None, :], axis=1, norm="forward").astype(T)
            else:
                yb = sfft.irfft(sfft.rfft(blk, axis=1) * filter_fd[None, :], n=nfft, axis=1, norm="forward").astype(T)
            o0 = save * (b_lo - 1 + r0)
            out[o0: o0 + yb.shape[0] * save] = yb[:, sv - 1:].reshape(-1)
        return out
    for bi in center_blocks:                    # :583-606
        data_offset = save * (bi - 1)
        data_stop = data_offset + save
        tdbuff = uT[data_offset - sv + 1: data_stop].copy()
        y = block(tdbuff)
        out[data_offset: data_stop] = y[sv - 1: nfft]
    return out


def conv_kern_fft(u, v, f64=False):
    """_conv_kern_fft!, src/dspbase.jl:611-644: one nextfastfft-sized FFT pair."""
    u = np.asarray(u)
    v = np.asarray(v)
    T = promote(u.dtype, v.dtype)
    if f64:
        T = np.dtype(np.complex128 if np.issubdtype(T, np.complexfloating) else np.float64)
    nout = len(u) + len(v) - 1
    nfft = nextfastfft(nout)
    up = np.zeros(nfft, dtype=T)
    up[:len(u)] = u
    vp = np.zeros(nfft, dtype=T)
    vp[:len(v)] = v
    if np.issubdtype(T, np.complexfloating):
        raw = sfft.ifft(sfft.fft(up) * sfft.fft(vp))
    else:
        raw = sfft.irfft(sfft.rfft(up) * sfft.rfft(vp), n=nfft)
    return raw[:nout].astype(T)


def conv_td(u, v):
    """_conv_td!, src/dspbase.jl:646-660: direct O(MN) muladd convolution in promote_type (exact for integers)."""
    u = np.asarray(u)
    v = np.asarray(v)
    if len(u) == 0 or len(v) == 0:
        return np.zeros(max(len(u) + len(v) - 1, 0), dtype=promote(u.dtype, v.dtype))
    return conv_td_nd(u, v)


def conv(u, v, algorithm="auto", f64=False):
    """conv(u, v; algorithm), 1-D: src/dspbase.jl:709-782 (algorithm resolution :720-743)."""
    u = np.asarray(u)
    v = np.asarray(v)
    T = promote(u.dtype, v.dtype)
    if algorithm == "auto":
        algorithm = "fast" if T.type in FFT_TYPES else "direct"
    if algorithm == "fast":
        algorithm = "direct" if len(u) * len(v) < 2 ** 16 else "fft"
    if algorithm == "direct" or len(u) == 0 or len(v) == 0:
        return conv_td(u, v)
    nout = len(u) + len(v) - 1
    small, large = (v, u) if len(u) >= len(v) else (u, v)
    os_nfft = optimalfftfiltlength(len(small), len(large))
    if algorithm == "fft":
        algorithm = "fft_overlapsave" if os_nfft < nout else "fft_simple"
    if algorithm == "fft_overlapsave":
        return conv_kern_os(large, small, os_nfft, f64=f64)
    if algorithm == "fft_simple":
        return conv_kern_fft(u, v, f64=f64)
    raise ValueError("algorithm must be :auto, :fast, :direct, :fft, :fft_simple, or :fft_overlapsave")


def conv_exact(u, v):
    """Ground truth: direct convolution in double precision (complex128/float64)."""
    u = np.asarray(u)
    v = np.asarray(v)
    W = np.complex128 if (np.iscomplexobj(u) or np.iscomplexobj(v)) else np.float64
    if len(u) * len(v) <= 1 << 24:
        return np.convolve(u.astype(W), v.astype(W))
    import scipy.signal as ss
    return ss.fftconvolve(u.astype(W), v.astype(W))


# --------------------------------------------------------------------------- N-D convolution (SURVEY.md 8f rank 4)

def conv_kern_fft_nd(u, v, f64=False):
    """_conv_kern_fft!, src/dspbase.jl:611-644, N-D: zero-pad both arrays to nextfastfft.(size(u) .+ size(v) .- 1), one
    rfft / fft pair over all dimensions, product, inverse, crop to the output size."""
    u = np.asarray(u)
    v = np.asarray(v)
    nd = max(u.ndim, v.ndim)
    u = u.reshape(u.shape + (1,) * (nd - u.ndim))          # rank promotion, :784-792
    v = v.reshape(v.shape + (1,) * (nd - v.ndim))
    T = promote(u.dtype, v.dtype)
    W = np.dtype(np.complex128 if np.issubdtype(T, np.complexfloating) else np.float64) if f64 else T
    oshape = tuple(a + b - 1 for a, b in zip(u.shape, v.shape))
    nffts = tuple(nextfastfft(n) for n in oshape)
    crop = tuple(slice(0, n) for n in oshape)
    if np.issubdtype(T, np.complexfloating):
        raw = sfft.ifftn(sfft.fftn(u.astype(W), nffts) * sfft.fftn(v.astype(W), nffts))
    else:
        # Julia's rfft halves the FIRST dimension; any real N-D transform gives the same product
        raw = sfft.irfftn(sfft.rfftn(u.astype(W), nffts) * sfft.rfftn(v.astype(W), nffts), nffts)
    return raw[crop].astype(W)


def conv_td_nd(u, v):
    """_conv_td!, src/dspbase.jl:646-660, N-D direct convolution in promote_type (exact for integers)."""
    u = np.asarray(u)
    v = np.asarray(v)
    nd = max(u.ndim, v.ndim)
    u = u.reshape(u.shape + (1,) * (nd - u.ndim))
    v = v.reshape(v.shape + (1,) * (nd - v.ndim))
    T = promote(u.dtype, v.dtype)
    u, v = u.astype(T), v.astype(T)
    out = np.zeros(tuple(a + b - 1 for a, b in zip(u.shape, v.shape)), dtype=T)
    # `for m in CartesianIndices(u), n in CartesianIndices(v)` when size(u,1) <= size(v,1), else n outer: the FIRST
    # iterator is the outer loop, and CartesianIndices run in column-major order (dim 1 fastest).  One step per outer
    # index adds that index's product to every output it reaches, so each output sums in the outer array's order.
    if u.shape[0] <= v.shape[0]:
        for m in (idx[::-1] for idx in np.ndindex(*u.shape[::-1])):
            sl = tuple(slice(i, i + n) for i, n in zip(m, v.shape))
            out[sl] = muladd(u[m], v, out[sl], T)
    else:
        for n in (idx[::-1] for idx in np.ndindex(*v.shape[::-1])):
            sl = tuple(slice(i, i + k) for i, k in zip(n, u.shape))
            out[sl] = muladd(u, v[n], out[sl], T)
    return out


def conv_kern_os_nd(u, v, nffts, f64=False):
    """unsafe_conv_kern_os!, src/dspbase.jl:490-609, with its perimeter blocks unsafe_conv_kern_os_edge!, :371-486, for
    arrays of any rank; `u` is the array with more elements (the caller orders them, :746-751), `nffts` one transform
    length per dimension.  Block by block as the reference: the time-domain buffer holds `nffts` samples that start
    `sv - 1` before the block's first output (zero where that lies outside `u`: pad_before / pad_after, :449-463), is
    transformed, multiplied by the filter spectrum (scaled once by 1/prod(nffts), :516), transformed back, and its valid
    region `sv : nffts` lands in `out` at `save_blocksize .* (block - 1)`, cropped where the output ends (:468-482).
    The centre blocks (:583-606) are the same statement with no padding, so one loop visits both kinds."""
    u = np.asarray(u)
    v = np.asarray(v)
    nd = u.ndim
    assert v.ndim == nd and len(nffts) == nd
    T = promote(u.dtype, v.dtype)
    W = np.dtype(np.complex128 if np.issubdtype(T, np.complexfloating) else np.float64) if f64 else T
    cplx = np.issubdtype(W, np.complexfloating)
    su, sv = u.shape, v.shape
    sout = tuple(a + b - 1 for a, b in zip(su, sv))
    nffts = tuple(int(n) for n in nffts)
    ideal = tuple(n - b + 1 for n, b in zip(nffts, sv))                       # :500
    deficit = tuple(max(0, i - s) for i, s in zip(ideal, sout))               # :503
    save = tuple(i - d for i, d in zip(ideal, deficit))                       # :505
    assert all(s >= 1 for s in save), "nffts must be at least size(v)"
    nblocks = tuple(-(-s // b) for s, b in zip(sout, save))                   # :506
    uW = u.astype(W)
    td = np.zeros(nffts, dtype=W)
    td[tuple(slice(0, n) for n in sv)] = v.astype(W)                          # _zeropad!(tdbuff, v), :513
    fwd = (lambda a: sfft.fftn(a)) if cplx else (lambda a: sfft.rfftn(a))
    inv = (lambda a: sfft.ifftn(a, norm="forward")) if cplx else (lambda a: sfft.irfftn(a, nffts, norm="forward"))
    filter_fd = fwd(td)
    filter_fd = (filter_fd * (1.0 / float(np.prod(nffts)))).astype(filter_fd.dtype)
    out = np.zeros(sout, dtype=W)
    for blk in np.ndindex(*nblocks):
        data_offset = tuple(s * b for s, b in zip(save, blk))                 # 0-based block index
        pad_before = tuple(max(0, b - o - 1) for b, o in zip(sv, data_offset))
        ideal_stop = tuple(o + s for o, s in zip(data_offset, save))
        pad_after = tuple(max(0, e - n) for e, n in zip(ideal_stop, su))
        lo = tuple(o - b + p + 1 for o, b, p in zip(data_offset, sv, pad_before))
        hi = tuple(e - p for e, p in zip(ideal_stop, pad_after))             # exclusive
        td = np.zeros(nffts, dtype=W)
        if all(h > l for h, l in zip(hi, lo)):
            td[tuple(slice(p, p + h - l) for p, h, l in zip(pad_before, hi, lo))] = uW[tuple(slice(l, h) for l, h in zip(lo, hi))]
        y = inv(fwd(td) * filter_fd).astype(W)                                # os_conv_block!, :337-356
        stop = tuple(min(o + s, n) for o, s, n in zip(data_offset, save, sout))
        cnt = tuple(e - o for e, o in zip(stop, data_offset))
        out[tuple(slice(o, e) for o, e in zip(data_offset, stop))] = y[tuple(slice(b - 1, b - 1 + c) for b, c in zip(sv, cnt))]
    return out
