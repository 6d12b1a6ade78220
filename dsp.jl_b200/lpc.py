"""Linear prediction, src/lpc.jl: lpc, arburg, levinson, LPCBurg, LPCLevinson.

Every call runs on the GPU (csrc/lpc.cu).  x may be the reference's host vector, a host len x nchan matrix or a
`DeviceArray` vector or matrix; each column of a matrix is one independent signal and every column runs in the same
launches (Burg: one, lpc Levinson: two, levinson: one).  Host inputs are copied to the device once and the results copied
back; `DeviceArray` inputs give `DeviceArray` results without a host synchronisation.  Integers compute in Float64 /
ComplexF64; the other eltypes in their own, `err` in the real eltype.

Everything but the reductions follows src/lpc.jl operation by operation; the reductions (dot(x, x), dot(eb, ef), the
autocorrelation lags) use the one fixed order of include/dspb200.h, which depends only on their length, so a column's result
does not depend on the other columns or on the kernel path.  The autocorrelation of lpc(x, p, LPCLevinson()) is a direct sum
over lags 0 .. p, not the reference's FFT xcorr (DESIGN.md section 4).
"""
import numpy as np

from . import _lib
from .clients import _DevWords
from .device import DeviceArray, to_device
from .dspbase import _gpu_dtype, _promote
from .errors import ArgumentError, BoundsError

LPC_P_MAX = 1024          # the library's largest order (shared-memory coefficient buffers)
_BURG, _LEVINSON = 0, 1


class LPCBurg:
    """Dispatch type of lpc: Burg's method (arburg), the default."""

    def __eq__(self, other):
        return isinstance(other, LPCBurg)

    def __hash__(self):
        return hash(LPCBurg)

    def __repr__(self):
        return "LPCBurg()"


class LPCLevinson:
    """Dispatch type of lpc: the biased autocorrelation and the Levinson recursion (levinson)."""

    def __eq__(self, other):
        return isinstance(other, LPCLevinson)

    def __hash__(self):
        return hash(LPCLevinson)

    def __repr__(self):
        return "LPCLevinson()"


def _order(p, what):
    if isinstance(p, (bool, np.bool_)) or not isinstance(p, (int, np.integer)):
        raise ArgumentError(f"{what}: the order p must be an integer")
    return int(p)


def _signal(x, what):
    """(x as a host array in its GPU eltype or the DeviceArray itself, rows, columns, host input?, vector input?)"""
    if isinstance(x, DeviceArray):
        if x.ndim not in (1, 2):
            raise ArgumentError(f"{what} takes a vector or a len x nchan matrix")
        return x, x.shape[0], (x.shape[1] if x.ndim == 2 else 1), False, x.ndim == 1
    x = np.asarray(x)
    if x.ndim not in (1, 2):
        raise ArgumentError(f"{what} takes a vector or a len x nchan matrix")
    G = _gpu_dtype(_promote(x))
    x = np.asfortranarray(x, dtype=G)
    return x, x.shape[0], (x.shape[1] if x.ndim == 2 else 1), True, x.ndim == 1


def _real(dt):
    return np.dtype(np.float32) if np.dtype(dt) in (np.float32, np.complex64) else np.dtype(np.float64)


def _check_p_max(p, what):
    if p > LPC_P_MAX:
        raise NotImplementedError(f"{what}: p = {p} exceeds LPC_P_MAX = {LPC_P_MAX}")


class _Call:
    """The device buffers of one call: the input on the device, the outputs a (na x ncols), err, refl (p x ncols or
    None) and the workspace."""

    def __init__(self, xx, host, n, ncols, p, na, want_refl, work_bytes):
        self.G = np.dtype(xx.dtype)
        self.xd = to_device(xx) if host else xx
        self.n, self.ncols, self.p = n, ncols, p
        self.a = DeviceArray((na, ncols), self.G)
        self.err = DeviceArray((ncols,), _real(self.G))
        self.refl = DeviceArray((p, ncols), self.G) if want_refl else None
        self.work = _DevWords(work_bytes, np.uint8) if work_bytes else None

    @property
    def refl_ptr(self):
        return None if self.refl is None else self.refl.ptr

    @property
    def work_ptr(self):
        return None if self.work is None else self.work.ptr


def _shape(d, host, vec, rows_from=0):
    """A (rows x ncols) DeviceArray result as the caller gets it: a host array or a DeviceArray, a vector / 0-d for a
    vector input; rows from `rows_from` on."""
    G = d.dtype
    rows, ncols = (d.shape[0], d.shape[1]) if d.ndim == 2 else (d.shape[0], 1)
    if d.ndim == 1:                                     # err
        if host:
            h = d.to_host()
            return h[0] if vec else h
        return DeviceArray((), G, _base=d, _ptr=d.ptr) if vec else d
    if host:
        h = d.to_host()[rows_from:]
        return h[:, 0].copy() if vec else h
    nr = rows - rows_from
    if vec:
        return DeviceArray((nr,), G, _base=d, _ptr=d.ptr + rows_from * G.itemsize)
    if rows_from == 0:
        return d
    out = DeviceArray((nr, ncols), G)
    if out.size:
        isz = G.itemsize
        _lib.memcpy2d_d2d(out.ptr, nr * isz, d.ptr + rows_from * isz, rows * isz, nr * isz, ncols)
    return out


def _burg(x, p, want_refl):
    xx, n, ncols, host, vec = _signal(x, "arburg")
    p = _order(p, "arburg")
    if p < 0 or p > n:
        raise ArgumentError(f"arburg needs 0 <= p <= length(x) (p = {p}, length {n})")
    _check_p_max(p, "arburg")
    c = _Call(xx, host, n, ncols, p, p + 1, want_refl, _lib.lpc_work_bytes(xx.dtype, n, ncols, p, _BURG) if ncols else 0)
    if ncols:
        _lib.lpc_burg_async(c.G, c.xd.ptr, n, ncols, p, c.a.ptr, c.err.ptr, c.refl_ptr, c.work_ptr)
    return c, host, vec


def _levinson_columns(x, p):
    xx, n, ncols, host, vec = _signal(x, "lpc")
    p = _order(p, "lpc")
    if p < 1 or p > n - 1:
        raise BoundsError(f"lpc(x, p, LPCLevinson()) needs 1 <= p <= length(x) - 1 (p = {p}, length {n})")
    _check_p_max(p, "lpc")
    c = _Call(xx, host, n, ncols, p, p, False, _lib.lpc_work_bytes(xx.dtype, n, ncols, p, _LEVINSON) if ncols else 0)
    if ncols:
        _lib.lpc_levinson_async(c.G, c.xd.ptr, n, ncols, p, c.a.ptr, c.err.ptr, None, c.work_ptr)
    return c, host, vec


def arburg(x, p):
    """arburg(x, p), src/lpc.jl:53-92: (a, prediction_err, reflection_coeffs) by Burg's method, a with its leading 1 and
    conjugated as the reference returns it.  For a len x nchan matrix: a is (p + 1) x nchan, err nchan, refl p x nchan.
    0 <= p <= length(x), else ArgumentError."""
    c, host, vec = _burg(x, p, True)
    return _shape(c.a, host, vec), _shape(c.err, host, vec), _shape(c.refl, host, vec)


def lpc(x, p, method=None):
    """lpc(x, p[, method]), src/lpc.jl:28-32, 94-98, 159: (a, prediction_err) without the leading 1; method LPCBurg()
    (the default) or LPCLevinson().  For a len x nchan matrix: a is p x nchan, err nchan."""
    if method is None or isinstance(method, LPCBurg):
        c, host, vec = _burg(x, p, False)
        return _shape(c.a, host, vec, rows_from=1), _shape(c.err, host, vec)
    if isinstance(method, LPCLevinson):
        c, host, vec = _levinson_columns(x, p)
        return _shape(c.a, host, vec), _shape(c.err, host, vec)
    raise ArgumentError(f"lpc: unknown method {method!r}; use LPCBurg() or LPCLevinson()")


def levinson(r, p):
    """levinson(R_xx, p), src/lpc.jl:122-146: (a, prediction_err, reflection_coeffs) from the autocorrelation r[0 .. p].
    r may be an nr x nchan matrix of autocorrelations (one column each).  1 <= p <= length(r) - 1, else BoundsError."""
    rr, nr, ncols, host, vec = _signal(r, "levinson")
    p = _order(p, "levinson")
    if p < 1 or p > nr - 1:
        raise BoundsError(f"levinson needs 1 <= p <= length(r) - 1 (p = {p}, length {nr})")
    _check_p_max(p, "levinson")
    c = _Call(rr, host, nr, ncols, p, p, True, 0)
    if ncols:
        _lib.levinson_async(c.G, c.xd.ptr, nr, ncols, p, c.a.ptr, c.err.ptr, c.refl.ptr)
    return _shape(c.a, host, vec), _shape(c.err, host, vec), _shape(c.refl, host, vec)
