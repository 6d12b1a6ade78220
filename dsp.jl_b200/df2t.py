"""PolynomialRatio and the stateful FIR filter DF2TFilter (src/Filters/coefficients.jl:66-216, src/Filters/filt.jl:17-30,
100-224, src/deprecated.jl:1-101), backed by the stateful instances of the tiled FIR kernel (dspb200_fir_exec_state*);
fftfilt(f::DF2TFilter, x) runs the same filter on the stateful overlap-save instances (dspb200_os_exec_state*).

In transposed direct form the FIR state is the partial multiply-add chain of the next nb - 1 outputs, so a signal
filtered block by block through one DF2TFilter gives bit-identical results to one call over the whole signal.  The GPU
path computes in one element type, the state's: it takes the combinations of coefficient, state and signal eltypes in
which the reference also computes every multiply-add in the state's eltype, and rejects the others before any work.
IIR coefficient sets (length(coefa) > 1) are outside the GPU scope and raise NotImplementedError.
"""
import numpy as np

from . import _lib
from .device import DeviceArray, to_device
from .dspbase import _cols
from .errors import ArgumentError, InexactError

_GPU_DTYPES = (np.dtype(np.float32), np.dtype(np.float64), np.dtype(np.complex64), np.dtype(np.complex128))


def _promote_type(*dts):
    """Julia's promote_type on numeric eltypes: integers and Bool give way to any floating-point type (Float32 and Int64
    promote to Float32, where numpy would pick float64); among floating-point types numpy agrees with Julia."""
    dts = [np.dtype(d) for d in dts]
    inexact = [d for d in dts if d.kind in "fc"]
    return np.result_type(*(inexact or dts))


def _real(dt):
    return np.dtype(np.float32) if np.dtype(dt) == np.complex64 else (
        np.dtype(np.float64) if np.dtype(dt) == np.complex128 else np.dtype(dt))


def _coef_z(v):
    """coef_z of the LaurentPolynomial the reference builds from v (highest power z^0 first): zeros at the oldest end
    are trimmed, an all-zero (or empty) vector becomes [0]; zeros at the z^0 end are kept (coef_z reads from z^0)."""
    nz = np.flatnonzero(v)
    return v[:nz[-1] + 1].copy() if nz.size else np.zeros(1, dtype=v.dtype)


class PolynomialRatio:
    """PolynomialRatio(b, a) in the z domain (src/Filters/coefficients.jl:95-150): eltype typeof(one(T1)/one(T2)),
    b and a divided by a[1]; `coefb` / `coefa` as coef_z returns them (src/Filters/coefficients.jl:195-216)."""

    def __init__(self, b, a):
        b = np.atleast_1d(np.asarray(b))
        a = np.atleast_1d(np.asarray(a))
        if b.ndim != 1 or a.ndim != 1:
            raise ArgumentError("PolynomialRatio takes coefficient vectors or numbers")
        if a.size == 0 or a[0] == 0:
            raise ArgumentError("filter must have non-zero leading denominator coefficient")
        T = _promote_type(b.dtype, a.dtype)
        if T.kind in "biu":                                  # Int / Int is Float64
            T = np.dtype(np.float64)
        a0 = a[0].astype(T) if a.dtype.kind == "c" else a[0].astype(_real(T))     # Complex / Real divides componentwise
        self.coefb = _coef_z((b.astype(T) / a0).astype(T))
        self.coefa = _coef_z((a.astype(T) / a0).astype(T))
        self.dtype = T

    def __repr__(self):
        return f"PolynomialRatio(coefb={self.coefb!r}, coefa={self.coefa!r})"


def coefb(f):
    return f.coefb


def coefa(f):
    return f.coefa


def _is_eltype(v):
    if isinstance(v, (np.dtype, type)):
        try:
            np.dtype(v)
            return True
        except TypeError:
            return False
    return False


class DF2TFilter:
    """DF2TFilter(coef, coldims), DF2TFilter(coef, sitype[, coldims]) and DF2TFilter(coef, si)
    (src/Filters/filt.jl:100-158) for FIR PolynomialRatio coefficients.  The state has nb - 1 rows and one column per
    channel (shape (nb - 1,) + coldims) and every `filt` call updates it.

    Residency is fixed at construction.  A host filter keeps `state` as a numpy array (the `si` passed in, as the
    reference keeps its array) and updates it in place.  An `si` that is a DeviceArray, or device=True, keeps the state in
    device memory: the filter takes DeviceArray chunks of the state's eltype, returns DeviceArrays and launches one kernel
    per non-empty chunk (fftfilt beyond the fused transform sizes: five per block batch and channel), alternating between
    two state buffers; `state` is the current one.  A DeviceArray `si` becomes
    the first of the two buffers, so after an odd number of calls it holds an older state: read `f.state`, not `si`.
    A device call cannot filter in place: `out` must not overlap `x` (the host filter can)."""

    def __init__(self, coef, *args, device=False):
        if not isinstance(coef, PolynomialRatio):
            raise NotImplementedError("DF2TFilter on the GPU takes PolynomialRatio coefficients; second-order sections, "
                                      "biquads and zero-pole-gain filters are outside the GPU scope")
        if coef.coefa.size > 1:
            raise NotImplementedError("IIR filtering (length(coefa) > 1) is outside the GPU hot-path scope (SURVEY.md 8a)")
        # the reference's methods (src/Filters/filt.jl:146-149); any other argument list is a MethodError there
        si_form = len(args) == 1 and not isinstance(args[0], tuple) and not _is_eltype(args[0])
        type_form = (len(args) >= 1 and _is_eltype(args[0]) and (len(args) == 1 or isinstance(args[1], tuple)))
        if len(args) > 2 or not (not args or si_form or type_form or (len(args) == 1 and isinstance(args[0], tuple))):
            raise TypeError("no method DF2TFilter(coef, " + ", ".join(type(a).__name__ for a in args) + "): the forms are "
                            "DF2TFilter(coef, coldims), DF2TFilter(coef, sitype[, coldims]) and DF2TFilter(coef, si)")
        self.coef = coef
        ns = max(coef.coefa.size, coef.coefb.size) - 1
        if si_form:
            si = args[0]
            self.device = isinstance(si, DeviceArray) or bool(device)
            if not isinstance(si, DeviceArray):
                si = np.asarray(si)
                if device:
                    si = to_device(si)
        else:
            V = coef.dtype
            coldims = ()
            if args and not isinstance(args[0], tuple):
                V = _promote_type(coef.dtype, np.dtype(args[0]))
                args = args[1:]
            if args:
                coldims = tuple(int(c) for c in args[0])
            si = np.zeros((ns,) + coldims, dtype=V)
            self.device = bool(device)
            if device:
                si = to_device(si)
        if len(si.shape) == 0 or si.shape[0] != ns:
            raise ArgumentError("length of state vector must match filter order")
        self._si = [si, DeviceArray(si.shape, si.dtype) if self.device else None]
        self._plan = None
        self._os = None

    @property
    def state(self):
        return self._si[0]

    @property
    def nstate(self):
        return self._si[0].shape[0]

    def _eltype(self, x_dtype):
        """The element type the kernel runs in (the state's); raises when the reference would compute otherwise."""
        S, X, C = np.dtype(self.state.dtype), np.dtype(x_dtype), self.coef.dtype
        if X.kind == "c" and S.kind != "c":
            raise InexactError("a complex signal cannot update a real filter state (InexactError in the reference)")
        P = _promote_type(C, S, X)
        if P != S:
            raise ArgumentError(f"the GPU DF2TFilter computes in the state's eltype: promote_type(coef {C}, state {S}, "
                                f"x {X}) = {P} differs from it, and the reference would round the state to {S} at every sample")
        if _real(_promote_type(C, X)) != _real(S):
            raise ArgumentError(f"the GPU DF2TFilter computes in the state's eltype {S}, but the reference forms the newest "
                                f"tap's product b[end]*x in the narrower {_promote_type(C, X)}")
        if S not in _GPU_DTYPES:
            raise ArgumentError(f"no GPU kernel for state eltype {S} (Float32, Float64, ComplexF32, ComplexF64)")
        return S

    def _fir_plan(self, S):
        if self._plan is None:
            self._plan = _lib.FirPlan(np.ascontiguousarray(self.coef.coefb, dtype=S))
        return self._plan

    def _os_plan(self, S):
        if self._os is None:
            self._os = _lib.OsPlan(np.ascontiguousarray(self.coef.coefb, dtype=S), 0)
        return self._os

    def _check_shapes(self, out, x):
        if tuple(x.shape) != tuple(out.shape):
            raise ArgumentError("out size must match x")
        if len(x.shape) == 0 or tuple(x.shape[1:]) != tuple(self.state.shape[1:]):
            raise ArgumentError("state size must match x")

    def filt(self, x):
        """filt(f::DF2TFilter, x), src/Filters/filt.jl:215-224: output eltype promote_type(eltype(state), eltype(x))."""
        return self._apply(x, self._fir_plan)

    def filt_(self, out, x):
        """filt!(out, f::DF2TFilter, x), src/Filters/filt.jl:157-181."""
        return self._apply_(out, x, self._fir_plan)

    def fftfilt(self, x):
        """fftfilt(f::DF2TFilter, x): the same stateful filter as filt(f, x), computed by overlap-save FFT convolution
        (dspb200_os_exec_state*).  The state is the same transposed direct-form state, so filt and fftfilt may alternate on
        one filter chunk by chunk.  filt is bit-identical to the reference's loop; fftfilt is within FFT rounding of it and
        costs about the same per output whatever the filter length.  Like the other GPU paths (and unlike the reference's
        real-only fftfilt) it takes Float32, Float64, ComplexF32 and ComplexF64, with filt's eltype rules."""
        return self._apply(x, self._os_plan)

    def fftfilt_(self, out, x):
        """fftfilt!(out, f::DF2TFilter, x): fftfilt(f, x) into out (see fftfilt)."""
        return self._apply_(out, x, self._os_plan)

    def _apply(self, x, plan):
        """filt / fftfilt: `plan(S)` is the plan whose exec_state / exec_state_dev runs the chunk."""
        if self.device:
            if not isinstance(x, DeviceArray):
                raise ArgumentError("a DF2TFilter with device-resident state filters DeviceArrays")
            S = self._eltype(x.dtype)
            return self._filt_device(DeviceArray(x.shape, S), x, S, plan)
        if isinstance(x, DeviceArray):
            raise ArgumentError("a DF2TFilter with host state filters host arrays (construct it with device=True)")
        x = np.asarray(x)
        S = self._eltype(x.dtype)
        return self._filt_host(np.empty(x.shape, dtype=S, order="F"), x, S, plan)

    def _apply_(self, out, x, plan):
        if self.device:
            if not (isinstance(x, DeviceArray) and isinstance(out, DeviceArray)):
                raise ArgumentError("a DF2TFilter with device-resident state filters DeviceArrays into DeviceArrays")
            S = self._eltype(x.dtype)
            if out.dtype != S:
                raise ArgumentError(f"out must have the state's eltype {S}")
            return self._filt_device(out, x, S, plan)
        if isinstance(x, DeviceArray) or isinstance(out, DeviceArray):
            raise ArgumentError("a DF2TFilter with host state filters host arrays (construct it with device=True)")
        x = np.asarray(x)
        S = self._eltype(x.dtype)
        if S.kind == "c" and np.dtype(out.dtype).kind != "c":
            raise InexactError(f"a {S} filter output cannot be stored in a real `out` (InexactError in the reference)")
        return self._filt_host(out, x, S, plan)

    def _filt_host(self, out, x, S, plan):
        self._check_shapes(out, x)
        nx = x.shape[0]
        ns = self.nstate
        if nx == 0 or x.size == 0:
            return out
        xS, nx, ncols = _cols(x, S)
        res = np.empty((nx, ncols), dtype=S, order="F")
        si = np.asfortranarray(self.state.reshape(ns, ncols), dtype=S) if ns else None
        so = np.empty((ns, ncols), dtype=S, order="F") if ns else None
        plan(S).exec_state(xS, nx, ncols, si, so, res)
        out[...] = res.reshape(x.shape)          # column c <-> trailing index c in C order, for x and the state alike
        if ns:
            self.state[...] = so.reshape(self.state.shape)
        return out

    def _filt_device(self, out, x, S, plan):
        self._check_shapes(out, x)
        if x.dtype != S:
            raise ArgumentError(f"device chunks must have the state's eltype {S} (got {x.dtype})")
        cur, nxt = self._si
        # the kernel's CTAs read the samples and state behind their neighbours' outputs: in place would race
        if out.overlaps(x) or out.overlaps(cur) or out.overlaps(nxt) or x.overlaps(nxt):
            raise ArgumentError("a device DF2TFilter cannot filter in place: out must not overlap x or the filter state")
        nx = x.shape[0]
        if nx == 0 or x.size == 0:
            return out
        plan(S).exec_state_dev(x.ptr, nx, x.size // nx, cur.ptr, nxt.ptr, out.ptr, 0)
        self._si = [nxt, cur]
        return out


def _deprecated_filter(coef, x, si):
    """The filter of the deprecated filt(b, a, x, si) / filt!(out, b, a, x, si) forms (src/deprecated.jl:1-30, 80-101):
    DF2TFilter(PolynomialRatio(b, a), copy(si)), a vector si repeated over the columns of x.  The caller's si is never
    modified."""
    if isinstance(x, DeviceArray) or isinstance(si, DeviceArray):
        raise ArgumentError("the filt(b, a, x, si) forms take host arrays; use a DF2TFilter for device-resident state")
    x = np.asarray(x)
    si = np.asarray(si)
    if si.ndim == 1 and x.ndim > 1:                       # repeat(si; outer=(1, size(x)[2:end]...))
        st = np.tile(si.reshape((-1,) + (1,) * (x.ndim - 1)), (1,) + x.shape[1:])
    else:
        st = si.copy()
    return DF2TFilter(coef, st), x


def filt_deprecated(b, a, x, si):
    f, x = _deprecated_filter(b if isinstance(b, PolynomialRatio) else PolynomialRatio(b, a), x, si)
    return f.filt(x)


def filt_deprecated_(out, b, a, x, si):
    f, x = _deprecated_filter(b if isinstance(b, PolynomialRatio) else PolynomialRatio(b, a), x, si)
    return f.filt_(out, x)
