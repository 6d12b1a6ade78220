"""Thin clients of the GPU convolution / FIR / FFT path (SURVEY.md 8f rank 3): xcorr, FIR filtfilt, finddelay,
shiftsignal, alignsignals, hilbert.  For host vectors each is a few host lines over `conv` / `filt_` / one FFT pair exactly
as in the reference.  Device-resident signals (`DeviceArray`) and channel matrices run every channel in one launch of the
same filter and correlation kernels, with the work around them -- the odd-symmetric extension, the peak search, the
shift -- in the kernels of csrc/clients.cu, so the samples never leave HBM."""
import ctypes as C

import numpy as np

from . import _lib
from .device import DeviceArray, _alloc, _release, sync, to_device
from .dspbase import SMALL_FILT_CUTOFF, _cols, _gpu_dtype, _os_plan, _promote, conv, optimalfftfiltlength
from .util import fftintype, fftouttype, nextfastfft
from .errors import ArgumentError, DimensionMismatch, DomainError
from .filters import filt_ as _filt_hx_


class _DevWords:
    """n device words of `itemsize` bytes (the int64 delays and int32 NaN flags of the peak search; DeviceArray holds only
    the four signal eltypes)."""

    def __init__(self, n, dtype):
        self.dtype = np.dtype(dtype)
        self.n = int(n)
        self._bytes = max(self.n * self.dtype.itemsize, 16)
        self.ptr = _alloc(self._bytes)

    def to_host(self):
        out = np.empty(self.n, dtype=self.dtype)
        if self.n:
            _lib.check(_lib.lib.dspb200_memcpy_d2h(_lib.ptr(out), self.ptr, self.n * self.dtype.itemsize, None))
            sync()
        return out

    def copy_from_host(self, a):
        a = np.ascontiguousarray(a, dtype=self.dtype)
        if self.n:
            _lib.check(_lib.lib.dspb200_memcpy_h2d(self.ptr, _lib.ptr(a), self.n * self.dtype.itemsize, None))
            sync()
        return self

    def __del__(self):
        try:
            if self.ptr:
                _release(self.ptr, self._bytes)
                self.ptr = 0
        except Exception:
            pass


def _keyword(k):
    return k.lstrip(":") if isinstance(k, str) else k


def _vector_on_host(v, what):
    """The shared vector of a column call, on the host (its conjugate-reverse becomes a filter, which plans take from the
    host): a DeviceArray vector is copied back."""
    if isinstance(v, DeviceArray):
        if v.ndim != 1:
            raise ArgumentError(f"{what} takes one vector as its second argument")
        return v.to_host()
    v = np.asarray(v)
    if v.ndim != 1:
        raise ArgumentError(f"{what} takes one vector as its second argument")
    return v


def _columns(x, what):
    """(array, rows, channels, host input?) of a DeviceArray vector / matrix or a host matrix."""
    if isinstance(x, DeviceArray):
        if x.ndim not in (1, 2):
            raise ArgumentError(f"{what} takes a vector or a len x nchan matrix")
        n = x.shape[0]
        return x, n, (x.shape[1] if x.ndim == 2 else 1), False
    x = np.asarray(x)
    if x.ndim != 2:
        raise ArgumentError(f"{what} takes a vector or a len x nchan matrix")
    return x, x.shape[0], x.shape[1], True


def _xcorr_route(nu, nv):
    """conv!'s chooser (src/dspbase.jl:720-743) for one column of nu samples against nv: :direct, :fft_overlapsave or
    :fft_simple."""
    if nu * nv < 2 ** 16:
        return "direct"
    nres = nu + nv - 1
    return "fft_overlapsave" if optimalfftfiltlength(min(nu, nv), max(nu, nv)) < nres else "fft_simple"


def _conv_columns(ud, nu, nchan, w, G):
    """conv(u[:, c], w) of every column of the device matrix ud (nu x nchan, eltype G) with the host vector w, on the route
    conv! picks for one column: the direct kernel (one launch), one overlap-save plan with w as the filter (every column in
    one fused launch), or one batched transform pair over the columns.  Returns the (nu + nw - 1) x nchan DeviceArray."""
    nv = w.size
    nres = nu + nv - 1
    out = DeviceArray((nres, nchan), G)
    if out.size == 0:
        return out
    w = np.ascontiguousarray(w, dtype=G)
    route = _xcorr_route(nu, nv)
    if route == "fft_overlapsave":
        _os_plan(w, None).exec_dev(ud.ptr, nu, nchan, out.ptr, nres, 0)
        return out
    dw = to_device(w)
    if route == "direct":
        _lib.conv_nd_dev(G, (nu, nchan), ud.ptr, (nv, 1), dw.ptr, None, out.ptr)
    else:
        _lib.conv_fft_columns(G, ud.ptr, nu, nchan, dw.ptr, nv, nextfastfft(nres), out.ptr)
    return out


def _xcorr_columns(u, v, padmode, scaling):
    """xcorr(u, v) of every column of a DeviceArray vector / matrix or a host matrix u with one vector v."""
    ux, nu, nchan, host = _columns(u, "xcorr")
    if v is None:
        if host or ux.ndim != 1:
            raise ArgumentError("xcorr of a matrix takes the vector v to correlate with")
        v = ux
    v = _vector_on_host(v, "xcorr")
    padmode, scaling = _keyword(padmode), _keyword(scaling)
    su, sv = nu, v.size
    if scaling == "biased" and su != sv:
        raise DimensionMismatch("scaling only valid for vectors of same length")
    if padmode not in ("none", "longest"):
        raise ArgumentError("padmode keyword argument must be either :none or :longest")
    if scaling not in ("none", "biased"):
        raise ArgumentError("scaling keyword argument must be either :none or :biased")
    T = _promote(ux, v)
    G = _gpu_dtype(T)
    if not host and T != ux.dtype:
        raise ArgumentError(f"xcorr of a DeviceArray computes in its eltype {ux.dtype}, but promote_type(u, v) is {T}")
    ud = to_device(np.asfortranarray(ux, dtype=G)) if host else ux
    if padmode == "longest" and su < sv:              # zero-pad every column to sv samples (one launch)
        padded = DeviceArray((sv, nchan), G)
        if padded.size:
            _lib.shift_async(G, ud.ptr, su, nchan, 0, None, False, padded.ptr, sv)
        ud, nu = padded, sv
    elif padmode == "longest" and sv < su:
        v = np.concatenate([v, np.zeros(su - sv, dtype=v.dtype)])
    w = np.conj(v)[::-1]                              # the host conjugate-reverse of xcorr(u, v) (src/dspbase.jl:896)
    out = _conv_columns(ud, nu, nchan, w, G)
    integer = np.dtype(T).kind in "biu"
    if scaling == "biased" and out.size and not integer:
        _lib.scale_div_async(G, out.ptr, out.size, su)
    if host:
        res = out.to_host()
        if integer:                                   # as the vector call: conv rounds to T, then res / su in Float64
            res = np.rint(res.real).astype(T)
            if scaling == "biased":
                res = res / su
        return res
    sync()
    if ux.ndim == 1:
        return DeviceArray((out.shape[0],), G, _base=out, _ptr=out.ptr)
    return out


def xcorr(u, v=None, padmode="none", scaling="none"):
    """xcorr(u[, v]; padmode, scaling), src/dspbase.jl:867-898: conv(u, reverse(conj(v))) -- conjugates the SECOND
    argument (MATLAB / scipy convention).

    Extension: u may be a `DeviceArray` vector or len x nchan matrix, or a host matrix, and v one vector on the host or the
    device.  Column c of the (nu + nv - 1) x nchan result is xcorr(u[:, c], v), all channels in one launch of the route
    conv! picks for one column: bit-identical to the vector call on :direct, and on :fft_overlapsave when v is the
    shorter argument (the vector call then makes v the filter too; when u is shorter it makes the column the filter, and
    the shared filter here rounds differently); :fft_simple runs one batched transform pair over the columns, within the
    convolution bound of DESIGN.md section 2.  A device u gives a DeviceArray, a host matrix a host array."""
    if isinstance(u, DeviceArray) or np.ndim(u) == 2:
        return _xcorr_columns(u, v, padmode, scaling)
    if isinstance(v, DeviceArray):
        v = _vector_on_host(v, "xcorr")
    return _xcorr_host(u, v, padmode, scaling)


def _xcorr_host(u, v=None, padmode="none", scaling="none"):
    u = np.asarray(u)
    v = u if v is None else np.asarray(v)
    if u.ndim != 1 or v.ndim != 1:
        raise ArgumentError("xcorr takes vectors")
    su, sv = u.size, v.size
    padmode = padmode.lstrip(":") if isinstance(padmode, str) else padmode
    scaling = scaling.lstrip(":") if isinstance(scaling, str) else scaling
    if scaling == "biased" and su != sv:
        raise DimensionMismatch("scaling only valid for vectors of same length")
    if padmode == "longest":
        if su < sv:
            u = np.concatenate([u, np.zeros(sv - su, dtype=u.dtype)])
        elif sv < su:
            v = np.concatenate([v, np.zeros(su - sv, dtype=v.dtype)])
    elif padmode != "none":
        raise ArgumentError("padmode keyword argument must be either :none or :longest")
    res = conv(u, np.conj(v)[::-1])
    if scaling == "biased":
        res = res / su
    elif scaling != "none":
        raise ArgumentError("scaling keyword argument must be either :none or :biased")
    return res


def _extrapolate_signal(sig, pad_length):
    """extrapolate_signal!, src/Filters/filt.jl:245-259: odd-symmetric extension of both ends."""
    n = sig.shape[0]
    # explicit indices: a slice stop of -1 (pad_length == n - 1, i.e. len(x) == len(b)) would mean "last element"
    head = 2 * sig[0] - sig[np.arange(pad_length, 0, -1)]
    tail = 2 * sig[n - 1] - sig[np.arange(n - 2, n - 2 - pad_length, -1)]
    return np.concatenate([head, sig, tail], axis=0)


def filtfilt(b, a_or_x, x=None):
    """filtfilt(b, x) / filtfilt(b, a, x) with length(a) == 1, src/Filters/filt.jl:301-337: zero-phase FIR filtering --
    the signal is extended odd-symmetrically by nb-1 samples and filtered once with conv(b, reverse(b)).

    A `DeviceArray` x (a vector or a len x nchan matrix, eltype promote_type(b, x)) is extended on the device for every
    channel in one launch, filtered by the kernel the host call picks (overlap-save for real data past 66 taps of
    conv(b, reverse(b)), else the time-domain FIR kernel) and cropped by a strided copy; the DeviceArray returned is
    bit-identical, column by column, to the host call."""
    b = np.asarray(b)
    dev = isinstance(a_or_x if x is None else x, DeviceArray)
    if x is None:
        x = a_or_x if dev else np.asarray(a_or_x)
    else:
        a = np.atleast_1d(np.asarray(a_or_x))
        x = x if dev else np.asarray(x)
        if a.size != 1:
            raise NotImplementedError("IIR filtfilt is outside the GPU hot-path scope (serial recurrence)")
        if a[0] != 1:
            b = b / a[0]
    if dev:
        return _filtfilt_device(b, x)
    nb = b.size
    if nb == 0:
        raise ArgumentError("filter vector b must be non-empty")
    if x.shape[0] < nb:
        raise ArgumentError("signal must be at least as long as the filter")     # BoundsError in the reference
    T = _promote(b, x)
    if T.kind in "biu":
        T = np.dtype(np.float64)
    bT = b.astype(T)
    newb = np.convolve(bT, bT[::-1])             # filt!(newb, b, reverse(b)) mirrored, :309-314 (2nb-1 taps, tiny, host)
    ext = _extrapolate_signal(x.astype(T), nb - 1)
    out = np.empty(ext.shape, dtype=T, order="F")
    _filt_hx_(out, newb.astype(T), ext)          # filt!(extrapolated, newb, extrapolated), :322
    return out[2 * nb - 2:]                       # drop garbage at start, :325


def _filtfilt_device(b, x):
    """filtfilt(b, x::DeviceArray): extrapolate_signal! in one launch, filt! of the extension with newb, the crop."""
    nb = b.size
    if nb == 0:
        raise ArgumentError("filter vector b must be non-empty")
    if x.ndim not in (1, 2):
        raise ArgumentError("filtfilt of a DeviceArray takes a vector or a len x nchan matrix")
    if x.shape[0] < nb:
        raise ArgumentError("signal must be at least as long as the filter")     # BoundsError in the reference
    T = _promote(b, x)
    if T != x.dtype:
        raise ArgumentError(f"filtfilt of a DeviceArray computes in its eltype {x.dtype}, but promote_type(b, x) is {T}")
    bT = b.astype(T)
    newb = np.ascontiguousarray(np.convolve(bT, bT[::-1]), dtype=T)   # :309-314, host design math as in the host call
    n, nchan, pad = x.shape[0], x.size // x.shape[0], nb - 1
    next_ = n + 2 * pad
    out = DeviceArray(x.shape, T)
    if nchan == 0:
        return out
    ext = DeviceArray((next_, nchan), T)
    _lib.filtfilt_extend_async(T, x.ptr, n, nchan, pad, ext.ptr)
    full = DeviceArray((next_, nchan), T)
    if T.kind == "f" and newb.size > SMALL_FILT_CUTOFF:          # filt_choose_alg!, src/Filters/filt.jl:537-555
        _os_plan(newb, None).exec_dev(ext.ptr, next_, nchan, full.ptr, next_, 0)
        plan = None
    else:
        plan = _lib.FirPlan(newb)
        plan.exec_dev(ext.ptr, next_, nchan, full.ptr, 0)
    isz = T.itemsize                                             # rows 2nb - 2 .. of every column, :325
    _lib.memcpy2d_d2d(out.ptr, n * isz, full.ptr + (2 * nb - 2) * isz, next_ * isz, n * isz, nchan)
    sync()
    if plan is not None:
        plan.close()
    return out


def _delays_dev(x, y):
    """The device half of finddelay(x, y) for the columns of x: (x on the device, its eltype, rows, channels, host input?,
    delays, NaN flags), the last two still being computed on the default stream.  The correlation is xcorr(x[:, c], y) with
    the shared reverse(y) as the filter -- xcorr(y, x)[k] == xcorr(x, y)[nres - 1 - k] for real data -- so every channel
    runs in one launch; the peak search reads it reversed."""
    xx, nx, nchan, host = _columns(x, "finddelay")
    y = _vector_on_host(y, "finddelay")
    if xx.dtype.kind == "c" or y.dtype.kind == "c":
        raise NotImplementedError("finddelay of a matrix or a DeviceArray takes real signals")
    T = _promote(xx, y)
    G = _gpu_dtype(T)
    if not host and T != xx.dtype:
        raise ArgumentError(f"finddelay of a DeviceArray computes in its eltype {xx.dtype}, but promote_type(x, y) is {T}")
    if nx == 0 or y.size == 0:
        raise ArgumentError("finddelay takes non-empty signals")
    xd = to_device(np.asfortranarray(xx, dtype=G)) if host else xx
    r = _conv_columns(xd, nx, nchan, y[::-1], G)
    delays, flags = _DevWords(nchan, np.int64), _DevWords(nchan, np.int32)
    if nchan:
        _lib.xcorr_peak_async(G, r.ptr, r.shape[0], nchan, nx, True, delays.ptr, flags.ptr)
    return xd, G, nx, nchan, host, delays, flags, r


def _delays_to_host(delays, flags):
    d = delays.to_host()                                     # the synchronisation that returns the delays
    if flags.to_host().any():
        raise ArgumentError("finddelay: a correlation holds a NaN (no maximum of |xcorr|)")
    return d


def finddelay(x, y):
    """finddelay(x, y), src/util.jl:360-368.

    Extension: x a len x nchan matrix (host or `DeviceArray`) or a DeviceArray vector, y one real reference vector (host
    or device): the delays of every column in one correlation launch and one peak-search launch, returned as an int64
    array (a Python int for a vector) after one synchronisation (and, on the :direct and :fft_simple routes, the wait
    at the end of the correlation).  The peak rule is the reference's (largest |xcorr|, then
    closest to the centre, then the lower index), applied to xcorr(x[:, c], y) read in reverse: its rounding differs from
    the vector call's xcorr(y, x), so on random data a near-tie may resolve differently; wherever the correlation is exact
    (integer data) the delays agree.  A column whose correlation holds a NaN raises ArgumentError."""
    if isinstance(x, DeviceArray) or np.ndim(x) == 2:
        xd, *_, delays, flags, _r = _delays_dev(x, y)
        d = _delays_to_host(delays, flags)
        return int(d[0]) if xd.ndim == 1 else d
    if isinstance(y, DeviceArray):
        y = _vector_on_host(y, "finddelay")
    x = np.asarray(x)
    y = np.asarray(y)
    s = xcorr(y, x, padmode="none")
    mag = np.abs(s)
    idxs = np.flatnonzero(mag == mag.max()) + 1          # 1-based like the reference
    center = x.size
    return int(center - idxs[np.argmin(np.abs(center - idxs))])


def shiftsignal(x, s):
    """shiftsignal(x, s), src/util.jl:379-412.

    A `DeviceArray` x (vector or len x nchan matrix) is shifted on the device, out of place, with zero fill; s is one
    integer or one integer per column.  DomainError when some |s| exceeds the length, before any launch."""
    if isinstance(x, DeviceArray):
        return _shiftsignal_device(x, s)
    x = np.array(x, copy=True)
    n = x.size
    if abs(s) > n:
        raise DomainError("The absolute value of s must not be greater than the length of x")
    if s > 0:
        x[s:] = x[:n - s].copy()
        x[:s] = 0
    elif s < 0:
        x[:n + s] = x[-s:].copy()
        x[n + s:] = 0
    return x


def _shiftsignal_device(x, s):
    if x.ndim not in (1, 2):
        raise ArgumentError("shiftsignal of a DeviceArray takes a vector or a len x nchan matrix")
    n = x.shape[0]
    nchan = x.shape[1] if x.ndim == 2 else 1
    per_column = np.ndim(s) == 1
    sv = np.asarray(s)
    if np.ndim(s) > 1 or sv.dtype.kind not in "iub" and not (sv.dtype.kind == "f" and np.all(sv == np.round(sv))):
        raise ArgumentError("shiftsignal takes an integer shift or one integer shift per column")
    sv = sv.astype(np.int64)
    if per_column and sv.size != nchan:
        raise DimensionMismatch(f"{sv.size} shifts for {nchan} columns")
    if np.any(np.abs(sv) > n):
        raise DomainError("The absolute value of s must not be greater than the length of x")
    out = DeviceArray(x.shape, x.dtype)
    if out.size == 0:
        return out
    if per_column:
        shifts = _DevWords(nchan, np.int64).copy_from_host(sv)
        _lib.shift_async(x.dtype, x.ptr, n, nchan, 0, shifts.ptr, False, out.ptr, n)
    else:
        _lib.shift_async(x.dtype, x.ptr, n, nchan, int(sv), None, False, out.ptr, n)
    sync()
    return out


def alignsignals(x, y):
    """alignsignals(x, y), src/util.jl:419-427.

    Extension, as finddelay: the columns of x (a host or `DeviceArray` matrix, or a DeviceArray vector) are shifted by
    minus their delays on the device, the shift reading the delays the peak search left in device memory, so the delays
    never visit the host between the peak search and the shift.  On the :fft_overlapsave route the correlation, peak search
    and shift are queued back to back and the one synchronisation returns d; on :direct and :fft_simple the correlation
    itself returns only once its work is done (cached plans and scratch, as every plan-less convolution), which is one
    more wait before the peak search is queued.  Returns (aligned, d): aligned a DeviceArray for a device x, a host array
    for a host matrix."""
    if isinstance(x, DeviceArray) or np.ndim(x) == 2:
        xd, G, nx, nchan, host, delays, flags, _r = _delays_dev(x, y)
        out = DeviceArray(xd.shape, G)
        if out.size:
            _lib.shift_async(G, xd.ptr, nx, nchan, 0, delays.ptr, True, out.ptr, nx)
        d = _delays_to_host(delays, flags)
        if np.any(np.abs(d) > nx):
            raise DomainError("The absolute value of s must not be greater than the length of x")
        if host:
            out = out.to_host()
        return out, (int(d[0]) if xd.ndim == 1 else d)
    d = finddelay(x, y)
    return shiftsignal(x, -d), d


def hilbert(x):
    """hilbert(x), src/util.jl:31-75: analytic signal x + j*H{x} of a real signal along the first dimension (every
    trailing index is an independent column).  Float32 stays single precision, every other real type is computed in
    Float64 (fftintype, src/util.jl:43, 92-94).  A `DeviceArray` is transformed in HBM and a `DeviceArray` returned."""
    if isinstance(x, DeviceArray):
        if x.dtype.kind != "f":
            raise ArgumentError("hilbert takes a real signal")
        n = x.shape[0] if x.ndim else 1
        ncols = x.size // max(n, 1)
        out = DeviceArray(x.shape, fftouttype(x.dtype))
        if x.size:
            _lib.hilbert_dev(x.dtype, x.ptr, n, ncols, out.ptr, 0)
        return out
    x = np.asarray(x)
    if x.dtype.kind == "c":
        raise ArgumentError("hilbert takes a real signal")
    tin = fftintype(x.dtype)
    a, n, ncols = _cols(x, tin)
    res = np.empty((n, ncols), dtype=fftouttype(tin), order="F")
    if a.size:
        _lib.hilbert(a, n, ncols, res)
    return res.reshape(x.shape)      # column c of res <-> trailing index c (C order over the trailing dims)
