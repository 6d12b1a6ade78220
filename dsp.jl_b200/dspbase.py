"""filt / conv front ends with the reference's signatures (src/dspbase.jl), backed by libdspb200.

Python spelling of the Julia names: `filt!` -> `filt_`, `conv!` -> `conv_`.  Arrays follow the reference's
column convention: axis 0 is time, all trailing axes are independent channels (src/dspbase.jl:55).
"""
import math

import numpy as np

from . import _lib
from .device import DeviceArray, to_device
from .errors import ArgumentError
from .util import nextfastfft

_OS_PLANS = {}          # small cache: (dtype, nfft, taps bytes) -> OsPlan (re-planning costs a filter transform)


def _os_plan(v, nfft):
    key = (v.dtype.str, int(nfft or 0), v.tobytes())
    plan = _OS_PLANS.get(key)
    if plan is None:
        if len(_OS_PLANS) >= 8:
            _OS_PLANS.pop(next(iter(_OS_PLANS))).close()
        plan = _OS_PLANS[key] = _lib.OsPlan(v, 0 if nfft is None else int(nfft))
    return plan

SMALL_FILT_CUTOFF = 66           # src/dspbase.jl:3
_FFT_DTYPES = (np.dtype(np.float32), np.dtype(np.float64), np.dtype(np.complex64), np.dtype(np.complex128))  # :674


def _promote(*arrs):
    dt = np.result_type(*[a.dtype if isinstance(a, DeviceArray) else np.asarray(a).dtype for a in arrs])
    if dt.kind in "biu":
        return dt
    if dt not in _FFT_DTYPES:            # float16, longdouble ... are outside the GPU path
        dt = np.dtype(np.complex128) if dt.kind == "c" else np.dtype(np.float64)
    return dt


def _gpu_dtype(dt):
    """Integers have no GPU kernels (SURVEY.md 8): compute in Float64 (exact for the reference's integer tests)."""
    dt = np.dtype(dt)
    return np.dtype(np.float64) if dt.kind in "biu" else dt


def _cols(x, dt):
    """Column-major (time fastest) contiguous copy/view of x in dtype dt; returns (array2d, nx, ncols)."""
    x = np.asarray(x)
    nx = x.shape[0] if x.ndim else 1
    a = np.asfortranarray(x.reshape(nx, -1), dtype=dt)
    return a, nx, a.shape[1]


# --------------------------------------------------------------------------------------------- filt(b, a, x)

def filt(b, a, x=None, si=None):
    """filt(b, a, x) (src/dspbase.jl:14-15) and, with two arguments, Filters.filt(h, x) (src/Filters/filt.jl:445-446),
    filt(f::DF2TFilter, x) and filt(f::PolynomialRatio, x) (src/Filters/filt.jl:30, 215-224).  The deprecated
    filt(b, a, x, si) and filt(f::PolynomialRatio, x, si) (src/deprecated.jl) filter from the initial state si (copied).
    filt(f::FIRFilter, x) streams x through the stateful polyphase filter (src/Filters/stream_filt.jl:627-637)."""
    from . import df2t
    from .filters import FIRFilter
    if isinstance(b, FIRFilter):
        if x is not None:
            raise ArgumentError("filt(f::FIRFilter, x) takes one signal")
        return b.filt(a)
    if isinstance(b, df2t.DF2TFilter):
        if x is not None:
            raise ArgumentError("filt(f::DF2TFilter, x) takes one signal")
        return b.filt(a)
    if isinstance(b, df2t.PolynomialRatio):
        if si is not None:
            raise ArgumentError("filt(f::PolynomialRatio, x, si) takes three arguments")
        if x is not None:
            return df2t.filt_deprecated(b, None, a, x)
        return filt(b.coefb, b.coefa, a)
    if si is not None:
        return df2t.filt_deprecated(b, a, x, si)
    if x is None:
        from .filters import filt as _filt_hx
        return _filt_hx(b, a)
    if isinstance(x, DeviceArray):
        return _filt_device(b, a, x)
    from fractions import Fraction
    if isinstance(x, (int, np.integer, Fraction)) and not isinstance(x, bool) and np.ndim(a) == 1 and np.ndim(b) == 1:
        from .filters import filt_multirate                     # filt(h, x, ratio), src/Filters/stream_filt.jl:663-666
        return filt_multirate(b, a, x)
    b = np.atleast_1d(np.asarray(b))
    a = np.atleast_1d(np.asarray(a))
    x = np.asarray(x)
    T = _promote(b, a, x)
    out = np.empty(x.shape, dtype=_gpu_dtype(T), order="F")
    filt_(out, b, a, x)
    return out      # integer inputs are computed and returned as Float64 (no integer GPU kernels)


def _filt_device(b, a, x):
    """filt(b, a, x::DeviceArray) with length(a) == 1: the same kernel as the host call, on the device-resident columns of
    x (its eltype must be promote_type(b, a, x)); returns a DeviceArray."""
    b = np.atleast_1d(np.asarray(b))
    a = np.atleast_1d(np.asarray(a))
    if b.size == 0:
        raise ArgumentError("filter vector b must be non-empty")
    if a.size == 0:
        raise ArgumentError("filter vector a must be non-empty")
    if a[0] == 0:
        raise ArgumentError("filter vector a[1] must be nonzero")
    if a.size != 1:
        raise NotImplementedError("IIR filtering (length(a) > 1) is outside the GPU hot-path scope (SURVEY.md 8a)")
    T = _promote(b, a, x)
    if T != x.dtype:
        raise ArgumentError(f"filt of a DeviceArray computes in its eltype {x.dtype}, but promote_type(b, a, x) is {T}")
    if a[0] != 1:                                   # :43-47 coefficient normalisation
        b = b / a[0]
    out = DeviceArray(x.shape, T)
    nx = x.shape[0] if x.ndim else 1
    if x.size:
        plan = _lib.FirPlan(np.ascontiguousarray(b, dtype=T))
        plan.exec_dev(x.ptr, nx, x.size // nx, out.ptr, 0)
        from .device import sync
        sync()
        plan.close()
    return out


def filt_(out, b, a, x=None, si=None):
    """filt!(out, b, a, x), src/dspbase.jl:26-66.  FIR only (length(a) == 1); IIR is outside the hot path.  Also
    filt!(out, f::DF2TFilter, x), filt!(out, f::PolynomialRatio, x) (src/Filters/filt.jl:17) and the deprecated
    filt!(out, b, a, x, si) / filt!(out, f::PolynomialRatio, x, si) (src/deprecated.jl, si copied).
    filt!(buffer, f::FIRFilter, x) returns the number of outputs written (src/Filters/stream_filt.jl:409-625)."""
    from . import df2t
    from .filters import FIRFilter
    if isinstance(b, FIRFilter):
        if x is not None:
            raise ArgumentError("filt!(buffer, f::FIRFilter, x) takes one signal")
        return b.filt_(out, a)
    if isinstance(b, df2t.DF2TFilter):
        if x is not None:
            raise ArgumentError("filt!(out, f::DF2TFilter, x) takes one signal")
        return b.filt_(out, a)
    if isinstance(b, df2t.PolynomialRatio):
        if si is not None:
            raise ArgumentError("filt!(out, f::PolynomialRatio, x, si) takes four arguments")
        if x is not None:
            return df2t.filt_deprecated_(out, b, None, a, x)
        return filt_(out, b.coefb, b.coefa, a)
    if si is not None:
        return df2t.filt_deprecated_(out, b, a, x, si)
    b = np.atleast_1d(np.asarray(b))
    a = np.atleast_1d(np.asarray(a))
    x = np.asarray(x)
    if b.size == 0:
        raise ArgumentError("filter vector b must be non-empty")
    if a.size == 0:
        raise ArgumentError("filter vector a must be non-empty")
    if a[0] == 0:
        raise ArgumentError("filter vector a[1] must be nonzero")
    if x.shape != out.shape:
        raise ArgumentError(f"output size {out.shape} must match input size {x.shape}")
    if a.size != 1:
        raise NotImplementedError("IIR filtering (length(a) > 1) is outside the GPU hot-path scope (SURVEY.md 8a)")
    if x.shape[0] == 0 if x.ndim else False:
        return out
    T = _gpu_dtype(_promote(b, a, x))
    if a[0] != 1:                                   # :43-47 coefficient normalisation
        b = b / a[0]
    bT = np.ascontiguousarray(b, dtype=T)
    xT, nx, ncols = _cols(x, T)
    res = np.empty((nx, ncols), dtype=T, order="F")
    plan = _lib.FirPlan(bT)
    plan.exec(xT, res)
    plan.close()
    out[...] = res.reshape(x.shape)      # column c of res <-> trailing index c (C order over the trailing dims)
    return out


# --------------------------------------------------------------------------------------------- planning

def os_fft_complexity(nfft, nb):
    """src/dspbase.jl:262."""
    return (nfft * math.log2(nfft) + nfft) / (nfft - nb + 1)


def optimalfftfiltlength(nb, nx):
    """src/dspbase.jl:268-291 (the reference's CPU cost model; kept for API parity and algorithm selection)."""
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


# --------------------------------------------------------------------------------------------- conv

_ALGORITHMS = ("auto", "fast", "direct", "fft", "fft_simple", "fft_overlapsave")


def conv(u, v, algorithm="auto", nfft=None):
    """conv(u, v; algorithm), src/dspbase.jl:775-782 (1-D).  `nfft` (extension) forces the overlap-save block
    transform length; by default the library picks the shared-memory size that suits the H100 kernel."""
    if isinstance(u, DeviceArray) or isinstance(v, DeviceArray):
        if isinstance(u, DeviceArray) and u.ndim == 1 and np.ndim(v) == 1 and not isinstance(v, DeviceArray):
            return _conv_device(u, v, algorithm, nfft)
        if not isinstance(algorithm, str):
            raise ArgumentError("conv(u, v, A) takes host arrays")
        if max(u.ndim, v.ndim) == 1:
            raise ArgumentError("1-D device convolution takes the long signal as a DeviceArray and the kernel as a host vector")
        return _conv_nd(u, v, algorithm)
    if not isinstance(algorithm, str):                        # conv(u, v, A): separable 2-D kernel, src/dspbase.jl:808-824
        return _conv_separable(u, v, algorithm)
    u = np.asarray(u)
    v = np.asarray(v)
    if u.ndim != 1 or v.ndim != 1:
        return _conv_nd(u, v, algorithm)
    T = _promote(u, v)
    out = np.empty(max(u.size + v.size - 1, 0), dtype=T)
    return conv_(out, u, v, algorithm=algorithm, nfft=nfft)


def _conv_nd(u, v, algorithm):
    """conv(u, v; algorithm) for arrays of rank 2 and 3 (and mixed ranks: the lower-rank argument gets trailing singleton
    dimensions, src/dspbase.jl:784-792).  Algorithm resolution as conv! (:720-751): `:fft_simple` is the single N-D
    transform pair of _conv_kern_fft! (:611-644); `:fft_overlapsave` the N-D blocking of unsafe_conv_kern_os! (:371-609)
    with the reference's block transforms optimalfftfiltlength.(size(small), size(large)) (:736); `:fft` picks
    overlap-save when a block transform is shorter than the output in some dimension (:737-743).  Either argument may be
    a DeviceArray (then both are taken to the device and the result stays there)."""
    if isinstance(algorithm, str) and algorithm.startswith(":"):
        algorithm = algorithm[1:]
    if algorithm not in _ALGORITHMS:
        raise ArgumentError("algorithm must be :auto, :fast, :direct, :fft, :fft_simple, or :fft_overlapsave")
    on_device = isinstance(u, DeviceArray) or isinstance(v, DeviceArray)
    nd = max(u.ndim, v.ndim)
    if nd > 3:
        raise NotImplementedError("convolution of arrays with more than 3 dimensions is outside the GPU scope")
    ushape = tuple(u.shape) + (1,) * (nd - u.ndim)
    vshape = tuple(v.shape) + (1,) * (nd - v.ndim)
    T = _promote(u, v)
    oshape = tuple(max(a + b - 1, 0) for a, b in zip(ushape, vshape))
    usize, vsize = int(np.prod(ushape)), int(np.prod(vshape))
    if usize == 0 or vsize == 0:                              # :730-731
        if on_device:
            raise ArgumentError("empty inputs are handled on the host path")
        return np.zeros(oshape, dtype=T)
    if algorithm == "auto":
        algorithm = "fast" if T in _FFT_DTYPES else "direct"
    if algorithm == "fast":
        algorithm = "direct" if usize * vsize < 2 ** 16 else "fft"
    swap = usize < vsize                                      # v should be the smaller array (:746-751)
    lshape, sshape = (vshape, ushape) if swap else (ushape, vshape)
    os_nffts = [optimalfftfiltlength(nb, nx) for nb, nx in zip(sshape, lshape)]      # :736
    if algorithm == "fft":                                    # :737-743
        algorithm = "fft_overlapsave" if any(n < o for n, o in zip(os_nffts, oshape)) else "fft_simple"
    overlapsave = algorithm == "fft_overlapsave"
    if algorithm == "direct":
        nffts = None
    elif overlapsave:
        nffts = os_nffts
    else:
        nffts = [nextfastfft(n) for n in oshape]
    G = _gpu_dtype(T)
    if on_device:
        du = u if isinstance(u, DeviceArray) else to_device(np.asarray(u, dtype=G))
        dv = v if isinstance(v, DeviceArray) else to_device(np.asarray(v, dtype=G))
        if du.dtype != G or dv.dtype != G:
            raise ArgumentError("device arguments of conv must share one floating-point eltype")
        if swap and overlapsave:
            du, dv, ushape, vshape = dv, du, vshape, ushape
        out = DeviceArray(oshape, G)
        _lib.conv_nd_dev(G, ushape, du.ptr, vshape, dv.ptr, nffts, out.ptr, overlapsave=overlapsave)
        return out
    uG = np.asfortranarray(np.asarray(u).reshape(ushape), dtype=G)
    vG = np.asfortranarray(np.asarray(v).reshape(vshape), dtype=G)
    if swap and overlapsave:
        uG, vG = vG, uG
    res = np.empty(oshape, dtype=G, order="F")
    _lib.conv_nd(uG, vG, nffts, res, overlapsave=overlapsave)
    if G == T:
        return res
    return np.rint(res).astype(T) if np.dtype(T).kind in "biu" else res.astype(T)     # integer inputs: exact in Float64


def _conv_separable(u, v, A):
    """conv(u, v, A), src/dspbase.jl:808-824: 2-D convolution of the matrix A with the separable kernel u * v' (computed by
    the reference with one 2-D FFT pair)."""
    u, v, A = np.asarray(u), np.asarray(v), np.asarray(A)
    if u.ndim != 1 or v.ndim != 1 or A.ndim != 2:
        raise ArgumentError("conv(u, v, A) takes two vectors and a matrix")
    T = _promote(u, v, A)
    G = np.dtype(np.float64) if np.dtype(T).kind in "biu" else _gpu_dtype(T)
    k = np.multiply.outer(u.astype(G), v.astype(G))
    return _conv_nd(A.astype(G), k, "fft_simple")


def _conv_device(u, v, algorithm, nfft):
    """conv(u::DeviceArray, v): the long signal stays in HBM; the (short) kernel v is a host vector.  Overlap-save only
    (the device pipeline form of `:fft_overlapsave`; `:auto/:fast/:fft` resolve to it for device inputs)."""
    v = np.ascontiguousarray(np.asarray(v), dtype=u.dtype)
    if u.ndim != 1 or v.ndim != 1:
        raise NotImplementedError("N-D convolution is outside the GPU hot-path scope (SURVEY.md 8a)")
    if algorithm not in ("auto", "fast", "fft", "fft_overlapsave"):
        raise ArgumentError("device inputs support algorithm :auto, :fast, :fft or :fft_overlapsave")
    if v.size == 0 or u.size == 0:
        raise ArgumentError("empty inputs are handled on the host path")
    if v.size > u.size:
        raise ArgumentError("the device-resident argument must be the longer one")
    nres = u.size + v.size - 1
    out = DeviceArray((nres,), u.dtype)
    _os_plan(v, nfft).exec_dev(u.ptr, u.size, 1, out.ptr, nres, 0)
    return out


def conv_(out, u, v, algorithm="auto", nfft=None):
    """conv!(out, u, v; algorithm), src/dspbase.jl:709-757 (1-D, non-offset axes)."""
    u = np.asarray(u)
    v = np.asarray(v)
    if isinstance(algorithm, str) and algorithm.startswith(":"):
        algorithm = algorithm[1:]
    T = _promote(u, v)
    nres = max(u.size + v.size - 1, 0)
    if out.ndim != 1 or out.size < nres:
        raise ArgumentError("out must be a vector of at least length(u)+length(v)-1 samples")
    if algorithm == "auto":                                   # :720-722
        algorithm = "fast" if T in _FFT_DTYPES else "direct"
    if algorithm == "fast":                                   # :723-729
        algorithm = "direct" if u.size * v.size < 2 ** 16 else "fft"
    if u.size == 0 or v.size == 0:                            # :730-731 -> _conv_td! zero-fills
        if algorithm not in _ALGORITHMS:
            raise ArgumentError("algorithm must be :auto, :fast, :direct, :fft, :fft_simple, or :fft_overlapsave")
        out[...] = 0
        return out
    G = _gpu_dtype(T)
    uG = np.ascontiguousarray(u, dtype=G)
    vG = np.ascontiguousarray(v, dtype=G)
    if algorithm == "direct":
        res = np.empty(nres, dtype=G)
        _lib.conv_direct(uG, vG, res)
    else:
        small, large = (vG, uG) if u.size >= v.size else (uG, vG)
        os_nfft = optimalfftfiltlength(small.size, large.size)   # :736
        if algorithm == "fft":                                # :737-743
            algorithm = "fft_overlapsave" if os_nfft < nres else "fft_simple"
        if algorithm == "fft_overlapsave":
            res = np.empty(nres, dtype=G)
            _os_plan(small, nfft).exec(large, res, large.size, 1, nres)
        elif algorithm == "fft_simple":
            res = np.empty(nres, dtype=G)
            _lib.conv_fft(uG, vG, nextfastfft(nres), res)       # :612-613
        else:
            raise ArgumentError("algorithm must be :auto, :fast, :direct, :fft, :fft_simple, or :fft_overlapsave")
    if out.dtype.kind in "biu" and res.dtype.kind in "fc":    # integer eltypes: round(Int, .) of the Float64 result (:775-776)
        res = np.rint(res.real)
    out[:nres] = res
    out[nres:] = 0                                            # :733-735 excess entries are zeroed
    return out
