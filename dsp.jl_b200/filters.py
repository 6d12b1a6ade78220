"""FIR application and polyphase resampling front ends (reference src/Filters/filt.jl:431-555,
src/Filters/stream_filt.jl, src/Filters/design.jl:547-559, 694-720), backed by libdspb200."""
import math
from collections import namedtuple
from fractions import Fraction

import numpy as np

from . import _lib
from .df2t import DF2TFilter
from .device import DeviceArray
from .dspbase import SMALL_FILT_CUTOFF, _cols, _gpu_dtype, _os_plan, _promote, filt_ as _filt_ba, optimalfftfiltlength
from .errors import ArgumentError, DomainError
from .windows import kaiser


# --------------------------------------------------------------------------------------------- tdfilt / fftfilt / filt(h, x)

def tdfilt(h, x):
    """tdfilt(h, x), src/Filters/filt.jl:431-433 -> filt(h, one(H), x)."""
    h = np.asarray(h)
    x = np.asarray(x)
    out = np.empty(x.shape, dtype=_gpu_dtype(_promote(h, x)), order="F")
    return tdfilt_(out, h, x)


def tdfilt_(out, h, x):
    """tdfilt!(out, h, x), src/Filters/filt.jl:441-443."""
    h = np.asarray(h)
    return _filt_ba(out, h, np.ones(1, dtype=h.dtype), x)


def _require_real(b, x):
    if np.iscomplexobj(b) or np.iscomplexobj(x):
        raise TypeError("fftfilt is defined for Real taps and Real signals only (src/Filters/filt.jl:458-459)")


def fftfilt(b, x, nfft=None):
    """fftfilt(b, x[, nfft]), src/Filters/filt.jl:458-461: real overlap-save along axis 0 of every column.
    nfft=None lets the library choose the block transform (the reference default is the CPU cost model
    optimalfftfiltlength); an explicit nfft is honoured.
    fftfilt(f::DF2TFilter, x) is the stateful form (DF2TFilter.fftfilt): filt(f, x) by overlap-save, carrying f's state."""
    if isinstance(b, DF2TFilter):
        if nfft is not None:
            raise ArgumentError("fftfilt(f::DF2TFilter, x) takes no nfft (the library chooses the block transform)")
        return b.fftfilt(x)
    b = np.asarray(b)
    if isinstance(x, DeviceArray):                       # device pipeline form: same-length overlap-save, stays in HBM
        if np.iscomplexobj(b) or x.dtype.kind == "c":
            raise TypeError("fftfilt is defined for Real taps and Real signals only (src/Filters/filt.jl:458-459)")
        nx = x.shape[0]
        out = DeviceArray(x.shape, x.dtype)
        if x.size:
            _os_plan(np.ascontiguousarray(b, dtype=x.dtype), nfft).exec_dev(x.ptr, nx, x.size // nx, out.ptr, nx, 0)
        return out
    x = np.asarray(x)
    _require_real(b, x)
    out = np.empty(x.shape, dtype=_gpu_dtype(_promote(b, x)), order="F")
    return _fftfilt(out, b, x, nfft)


def fftfilt_(out, b, x, nfft=None):
    """fftfilt!(out, b, x[, nfft]), src/Filters/filt.jl:468-476; fftfilt!(out, f::DF2TFilter, x) is the stateful form."""
    if isinstance(b, DF2TFilter):
        if nfft is not None:
            raise ArgumentError("fftfilt!(out, f::DF2TFilter, x) takes no nfft (the library chooses the block transform)")
        return b.fftfilt_(out, x)
    b = np.asarray(b)
    x = np.asarray(x)
    _require_real(b, x)
    if out.shape != x.shape:
        raise ArgumentError("out and x must be the same size")
    return _fftfilt(out, b, x, nfft)


def _fftfilt(out, b, x, nfft):
    """_fftfilt!, src/Filters/filt.jl:479-521 (the block loop runs on the GPU)."""
    if b.size == 0:
        raise ArgumentError("filter vector b must be non-empty")
    W = _gpu_dtype(_promote(b, x))
    if x.size == 0:
        return out
    xW, nx, ncols = _cols(x, W)
    bW = np.ascontiguousarray(b, dtype=W)
    if nfft is not None and nfft < b.size:
        raise ArgumentError("nfft must be >= length(b)")     # the reference leaves this unchecked (garbage result)
    res = np.empty((nx, ncols), dtype=W, order="F")
    _os_plan(bW, nfft).exec(xW, res, nx, ncols, nx)
    out[...] = res.reshape(x.shape)
    return out


def filt(b, x):
    """filt(b, x), src/Filters/filt.jl:445-446, 525-527."""
    b = np.asarray(b)
    x = np.asarray(x)
    out = np.empty(x.shape, dtype=_gpu_dtype(_promote(b, x)), order="F")
    return _filt_choose_alg(out, b, x)


def filt_(out, b, x):
    """filt!(out, b, x), src/Filters/filt.jl:530-533."""
    b = np.asarray(b)
    x = np.asarray(x)
    if out.shape != x.shape:
        raise ArgumentError("out must be the same size as x")
    return _filt_choose_alg(out, b, x)


def _filt_choose_alg(out, b, x):
    """filt_choose_alg!, src/Filters/filt.jl:537-555: Real x Real with nb > 66 -> overlap-save, else time domain."""
    real = not (np.iscomplexobj(b) or np.iscomplexobj(x))
    if real and b.size > SMALL_FILT_CUTOFF:
        return _fftfilt(out, b, x, None)
    return tdfilt_(out, b, x)


# --------------------------------------------------------------------------------------------- default taps

def kaiserord(transitionwidth, attenuation=60):
    """src/Filters/design.jl:547-559."""
    n = math.ceil((attenuation - 7.95) / (math.pi * 2.285 * transitionwidth)) + 1
    if attenuation > 50:
        beta = 0.1102 * (attenuation - 8.7)
    elif attenuation >= 21:
        beta = 0.5842 * (attenuation - 21) ** 0.4 + 0.07886 * (attenuation - 21)
    else:
        beta = 0.0
    return n, beta / math.pi


def _resample_filter(f_nyq, nphi, rel_bw, attenuation):
    """_resample_filter, src/Filters/design.jl:701-720: Kaiser-windowed sinc lowpass, length rounded up to an odd multiple
    of Nphi, DC gain Nphi."""
    cutoff = f_nyq * rel_bw
    hlen, alpha = kaiserord(cutoff * 0.2, attenuation)
    hlen = nphi * math.ceil(hlen / nphi)
    hlen += (hlen % 2 == 0)
    k = np.arange(1, hlen + 1, dtype=np.float64)
    h = cutoff * np.sinc(cutoff * (k - (hlen + 1) / 2)) * kaiser(hlen, alpha)   # :598-602, FIRWindow :669-674
    h *= 1 / h.sum()                                                              # scalefactor(Lowpass) :642
    return h * nphi                                                               # rmul!(h, Nphi) :719


def resample_filter(rate, *args):
    """resample_filter(rate::Union{Integer,Rational}, rel_bw=1.0, attenuation=60) (src/Filters/design.jl:694-699) and
    resample_filter(rate::AbstractFloat, Nphi=32, rel_bw=1.0, attenuation=60) (:683-686)."""
    if isinstance(rate, (float, np.floating)):
        nphi, rel_bw, attenuation = (list(args) + [32, 1.0, 60][len(args):])[:3]
        nphi = int(nphi)
        return _resample_filter(1.0 / nphi if rate >= 1.0 else rate / nphi, nphi, rel_bw, attenuation)
    rel_bw, attenuation = (list(args) + [1.0, 60][len(args):])[:2]
    rate = _as_ratio(rate)
    nphi, dec = rate.numerator, rate.denominator
    return _resample_filter(min(1 / nphi, 1 / dec), nphi, rel_bw, attenuation)


def _as_ratio(rate):
    if isinstance(rate, (float, np.floating)):
        raise ArgumentError("a floating-point rate selects the arbitrary-rate (FIRArbitrary) path; pass an int or "
                            "fractions.Fraction here")
    if isinstance(rate, str):
        rate = rate.replace("//", "/")
    return Fraction(rate)


def _round_half_even(v):
    return int(np.round(v))     # Julia's round(Int, x) is ties-to-even


def resample_phase(hlen, rate):
    """undelay! -> setphase!(timedelay): src/Filters/stream_filt.jl:216-229, 400-403, 706-714.
    Returns (n0, phi0): input samples skipped and 0-based start phase."""
    I, D = rate.numerator, rate.denominator
    if I == 1:                                    # FIRStandard / FIRDecimator: tau = (hLen-1)/2, whole samples only
        return _round_half_even((hlen - 1) / 2), 0
    tau = (hlen - 1) / (2 * I)
    q, r = divmod(_round_half_even(tau * I), I)
    return q, r


# --------------------------------------------------------------------------------------------- FIRFilter (stateful)

def outputlength(inputlength_, ratio, initial_phi):
    """outputlength(inputlength, ratio, initialphi), src/Filters/stream_filt.jl:317-322 (initialphi is 1-based)."""
    ratio = _as_ratio(ratio)
    return -((-(inputlength_ * ratio.numerator - initial_phi + 1)) // ratio.denominator)


def inputlength(outputlength_, ratio, initial_phi, round_up=False):
    """inputlength(outputlength, ratio, initialphi, RoundDown | RoundUp), src/Filters/stream_filt.jl:358-364."""
    ratio = _as_ratio(ratio)
    d = ratio.denominator if round_up else 1
    num = outputlength_ * ratio.denominator + initial_phi - d
    return -((-num) // ratio.numerator) if round_up else num // ratio.numerator


_Step = namedtuple("_Step", "nout n0 phase0 j_seam phi_idx input_deficit phi_accumulator")


class FIRFilter:
    """FIRFilter(h, ratio=1): stateful single-rate / interpolating / decimating / rational polyphase FIR filter,
    src/Filters/stream_filt.jl:137-178 (kernels :8-78).  State carried across `filt` calls exactly as the
    reference: `history` (last historyLen input samples), `phi_idx` (1-based phase) and `input_deficit`
    (:476-515).  Each call runs the polyphase kernel on [history; x] through the closed form of the phase
    recurrence.

    FIRFilter(h, rate::float, nphases=32) is the arbitrary-rate filter (FIRArbitrary, :92-134, 193-205): polyphase bank
    plus derivative bank with linear interpolation between phases; state `phi_accumulator` / `input_deficit`.  The
    per-call phase sequence acc0 + j*delta is evaluated exactly (rational arithmetic on the host for the counts,
    double-double on the device), see resample.cu.  `h=None` designs the taps with resample_filter(rate, nphases).

    device=True keeps the history in device memory: the filter takes DeviceArray chunks, a vector (nx,) or a column-major
    (nx, nchan) matrix whose channels share the one phase state (an extension: the reference filters vectors), and
    returns DeviceArrays.  A chunk costs at most two kernel launches, no host synchronisation and no host <-> device
    copy; the kernels read the virtual column [history; x] without building it.  The first chunk fixes the eltype and
    the channel count; `reset()` drops them with the history.  `history` is then the current (tpp - 1)-sample device
    buffer (None before the first launch).  A host filter refuses DeviceArrays and a device filter host arrays."""

    def __init__(self, h, ratio=1, nphases=32, *, device=False):
        self.device = bool(device)
        if isinstance(ratio, (float, np.floating)):
            self._init_arbitrary(h, float(ratio), int(nphases))
            return
        self.ratio = _as_ratio(ratio)
        if self.ratio <= 0:
            raise ArgumentError("ratio must be positive")
        h = np.asarray(h)
        if h.ndim != 1 or h.size == 0:
            raise ArgumentError("h must be a non-empty vector")
        if np.iscomplexobj(h):
            raise NotImplementedError("complex taps are outside the GPU hot-path scope")
        self.h = np.ascontiguousarray(h, dtype=np.float32 if h.dtype == np.float32 else np.float64)
        self.interpolation, self.decimation = self.ratio.numerator, self.ratio.denominator
        self.hlen = self.h.size
        I, D = self.interpolation, self.decimation
        if self.ratio == 1:
            self.kind, self.history_len = "standard", self.hlen - 1
        elif D == 1:
            self.kind, self.history_len = "interpolator", -(-self.hlen // I) - 1
        elif I == 1:
            self.kind, self.history_len = "decimator", self.hlen - 1
        else:
            self.kind, self.history_len = "rational", -(-self.hlen // I) - 1
        self.taps_per_phase = -(-self.hlen // I)
        self._plans = {}
        self.reset()

    def _init_arbitrary(self, h, rate, nphases):
        if not rate > 0.0:
            raise DomainError("rate must be greater than 0")                                  # :194
        if h is None:
            h = resample_filter(rate, nphases)
        h = np.asarray(h)
        if h.ndim != 1 or h.size == 0:
            raise ArgumentError("h must be a non-empty vector")
        if np.iscomplexobj(h):
            raise NotImplementedError("complex taps are outside the GPU hot-path scope")
        self.h = np.ascontiguousarray(h, dtype=np.float32 if h.dtype == np.float32 else np.float64)
        self.kind, self.rate, self.nphases = "arbitrary", rate, nphases
        self.ratio = rate
        self.hlen = self.h.size
        self.taps_per_phase = -(-self.hlen // nphases)
        self.history_len = self.taps_per_phase - 1
        self.delta = nphases / rate                                                           # :115
        self._plans = {}
        self.reset()

    def reset(self):
        """reset!, src/Filters/stream_filt.jl:247-276.  A device filter also drops its history buffers, eltype and
        channel count."""
        self.phi_idx = 1
        self.input_deficit = 1
        self.history = None
        self.phi_accumulator = 0.0
        self._dev_key = None          # device form: (eltype, channel shape) fixed by the first chunk
        self._hist = None             # device form: [current, next] history buffers
        return self

    @property
    def alpha(self):
        return math.modf(self.phi_accumulator)[0]

    def timedelay(self):
        """timedelay, src/Filters/stream_filt.jl:400-403."""
        if self.kind == "arbitrary":
            return (self.hlen - 1) / (2 * self.nphases)
        if self.kind in ("rational", "interpolator"):
            return (self.hlen - 1) / (2 * self.interpolation)
        return (self.hlen - 1) / 2

    def setphase(self, phi):
        """setphase!, src/Filters/stream_filt.jl:216-229."""
        if phi < 0:
            raise DomainError("phi must be >= 0")
        if self.kind == "arbitrary":                                                          # :231-239
            frac, whole = math.modf(phi)
            self.input_deficit += _round_half_even(whole)
            self.phi_accumulator = frac * self.nphases
            self.phi_idx = 1 + math.floor(self.phi_accumulator)
        elif self.kind in ("rational", "interpolator"):
            q, r = divmod(_round_half_even(phi * self.interpolation), self.interpolation)
            self.input_deficit += q
            self.phi_idx = r + 1
        else:
            self.input_deficit += _round_half_even(phi)

    def outputlength(self, inlen):
        """outputlength(::FIRFilter, inputlength), src/Filters/stream_filt.jl:324-342."""
        if self.kind == "standard":
            return inlen
        if self.kind == "arbitrary":                                                          # :340-342
            return math.ceil((inlen - self.input_deficit + 1) * self.rate - self.phi_accumulator / self.delta)
        return outputlength(inlen - self.input_deficit + 1, self.ratio, self.phi_idx if self.kind != "decimator" else 1)

    def inputlength(self, outlen, round_up=False):
        """inputlength(::FIRFilter, outputlength, r), src/Filters/stream_filt.jl:366-398."""
        if self.kind == "standard":
            return outlen
        if self.kind == "arbitrary":                                                          # :385-389
            d = 1 if round_up else 0
            return math.floor((outlen - d + self.phi_accumulator / self.delta) / self.rate) + d + self.input_deficit - 1
        v = inputlength(outlen, self.ratio, self.phi_idx if self.kind != "decimator" else 1, round_up)
        return v + self.input_deficit - 1

    def _step(self, phi_idx, input_deficit, phi_accumulator, xlen):
        """Bookkeeping of one filt! call on xlen samples from the state (phi_idx, input_deficit, phi_accumulator), shared by
        the host and the device form (src/Filters/stream_filt.jl:476-515, 522-560, 579-625).  Returns a _Step: `nout`
        outputs; `n0`, the index in [history; x] of output 0's newest sample; `phase0`, the 0-based start phase (rational
        kinds) or the phase accumulator (arbitrary); `j_seam`, the number of outputs whose window reaches into the history
        (rational kinds; the arbitrary-rate kernel reads [history; x] itself, so 0 there); and the state after the call.
        Output j's oldest sample in [history; x] is input_deficit - 1 + (phase0 + j*D) // I, so it reads the history iff
        (phase0 + j*D) // I < history_len - input_deficit + 1."""
        H = self.history_len
        n0 = H + input_deficit - 1
        if xlen < input_deficit:                                                              # :484-488, :590-594
            return _Step(0, n0, phi_accumulator if self.kind == "arbitrary" else 0, 0, phi_idx, input_deficit - xlen,
                         phi_accumulator)
        if self.kind == "arbitrary":
            nout, deficit, acc = _arb_advance(phi_accumulator, input_deficit, self.delta, self.nphases, xlen)
            return _Step(nout, n0, phi_accumulator, 0, 1 + math.floor(acc), deficit, acc)
        I, D = self.interpolation, self.decimation
        phased = self.kind in ("rational", "interpolator")
        phi0 = phi_idx - 1 if phased else 0
        nout = outputlength(xlen - input_deficit + 1, self.ratio, phi0 + 1) if self.kind != "standard" else xlen
        total = phi0 + nout * D                                            # phase recurrence after nout outputs
        deficit = 1 if self.kind == "interpolator" else input_deficit + total // I - xlen     # :463, :511
        K = H - input_deficit + 1
        j_seam = min(nout, -(-(I * K - phi0) // D)) if K > 0 and I * K > phi0 else 0
        return _Step(nout, n0, phi0, j_seam, total % I + 1 if phased else phi_idx, deficit, phi_accumulator)

    def _commit(self, st):
        self.phi_idx, self.input_deficit, self.phi_accumulator = st.phi_idx, st.input_deficit, st.phi_accumulator

    def _plan(self, xdt):
        if xdt not in self._plans:
            self._plans[xdt] = (_lib.ResampleArbPlan(xdt, self.h, self.nphases) if self.kind == "arbitrary"
                                else _lib.ResamplePlan(xdt, self.h, self.interpolation, self.decimation))
        return self._plans[xdt]

    def filt(self, x):
        """filt(self::FIRFilter, x), src/Filters/stream_filt.jl:627-637 (+ the filt! loops :409-560)."""
        if self.device:
            return self._filt_device(None, x)
        return self._filt_host(x)[0]

    def filt_(self, buffer, x):
        """filt!(buffer, self::FIRFilter, x), src/Filters/stream_filt.jl:409-625: writes the call's outputs to the first
        elements of `buffer` (its first `nout` rows for a device matrix) and returns their number.  A buffer shorter than
        the call's output raises ArgumentError before the state changes; so does, for a device filter, a buffer that
        overlaps x."""
        if self.device:
            return self._filt_device(buffer, x)
        if isinstance(buffer, DeviceArray):
            raise ArgumentError("a host FIRFilter filters host arrays (construct it with device=True)")
        return self._filt_host(x, buffer)[1]

    def _filt_host(self, x, buffer=None):
        if isinstance(x, DeviceArray):
            raise ArgumentError("a host FIRFilter filters host arrays (construct it with device=True)")
        x = np.asarray(x)
        if x.ndim != 1:
            raise ArgumentError("FIRFilter filters vectors")
        xdt = _gpu_dtype(_promote(x))
        x = np.ascontiguousarray(x, dtype=xdt)
        xlen = x.size
        st = self._step(self.phi_idx, self.input_deficit, self.phi_accumulator, xlen)
        if buffer is not None and len(buffer) < st.nout:
            raise ArgumentError(f"buffer is too small: the call produces {st.nout} outputs, buffer holds {len(buffer)}")
        plan = self._plan(xdt)
        if self.history is None or self.history.dtype != xdt:
            self.history = np.zeros(self.history_len, dtype=xdt)          # history = zeros(historyLen), :175
        if xlen < self.input_deficit:                                      # :484-488, :590-594
            self.history = self._shiftin(self.history, x)
            self._commit(st)
            return np.zeros(0, dtype=plan.out_dtype), 0
        xe = np.concatenate([self.history, x])
        out = np.empty(st.nout, dtype=plan.out_dtype)
        if self.kind == "arbitrary":                                       # :579-625
            plan.exec(xe, xe.size, st.n0, st.phase0, self.delta, out, st.nout)
        else:
            plan.exec(xe, xe.size, 1, st.n0, st.phase0, out, st.nout)
        self._commit(st)
        self.history = self._shiftin(self.history, x)                      # :512, :621
        if buffer is not None:
            buffer[:st.nout] = out
        return out, st.nout

    def _filt_device(self, buffer, x):
        """One chunk through dspb200_resample_(arb_)stream_exec_dev: every check happens before the first launch."""
        if not isinstance(x, DeviceArray):
            raise ArgumentError("a device FIRFilter filters DeviceArrays (construct it without device=True for host arrays)")
        if x.ndim not in (1, 2):
            raise ArgumentError("a device FIRFilter filters a vector or a len x nchan DeviceArray")
        key = (x.dtype, x.shape[1:])
        if self._dev_key is not None and key != self._dev_key:
            raise ArgumentError(f"this device FIRFilter streams {self._dev_key[0]} chunks of channel shape {self._dev_key[1]}; "
                                f"got {x.dtype} {x.shape[1:]} (reset() starts a new stream)")
        plan = self._plan(x.dtype)
        nx = x.shape[0]
        nchan = x.shape[1] if x.ndim == 2 else 1
        st = self._step(self.phi_idx, self.input_deficit, self.phi_accumulator, nx)
        hshape = (self.history_len,) + x.shape[1:]
        hist = self._hist or [None, DeviceArray(hshape, x.dtype)]

        if buffer is None:
            out = DeviceArray((st.nout,) + x.shape[1:], plan.out_dtype)
        else:
            if not isinstance(buffer, DeviceArray):
                raise ArgumentError("a device FIRFilter writes into a DeviceArray buffer")
            if buffer.dtype != plan.out_dtype or buffer.shape[1:] != x.shape[1:]:
                raise ArgumentError(f"buffer must be a {plan.out_dtype} DeviceArray of channel shape {x.shape[1:]}")
            if buffer.shape[0] < st.nout:
                raise ArgumentError(f"buffer is too small: the call produces {st.nout} outputs, buffer holds {buffer.shape[0]}")
            if buffer.overlaps(x) or buffer.overlaps(hist[0]) or buffer.overlaps(hist[1]):
                raise ArgumentError("a device FIRFilter cannot filter in place: buffer must not overlap x")
            out = buffer
        if self._hist is None:
            self._dev_key, self._hist = key, hist
        if nx and nchan:
            cur, nxt = hist
            ldo = out.shape[0]
            if self.kind == "arbitrary":
                plan.stream_exec_dev(cur.ptr if cur is not None else None, nxt.ptr, x.ptr, nx, nchan, self.input_deficit,
                                     st.phase0, self.delta, out.ptr, ldo, st.nout, 0)
            else:
                plan.stream_exec_dev(cur.ptr if cur is not None else None, nxt.ptr, x.ptr, nx, nchan, self.input_deficit,
                                     st.phase0, out.ptr, ldo, st.nout, 0)
            if cur is None:                                                # the first launch: zero history in, none to reuse
                cur = DeviceArray(hshape, x.dtype)
            self._hist = [nxt, cur]
            self.history = nxt
        self._commit(st)
        return out if buffer is None else st.nout

    @staticmethod
    def _shiftin(a, b):
        """shiftin!, src/util.jl:299-314."""
        if a.size == 0:
            return a
        return np.concatenate([a, b.astype(a.dtype, copy=False)])[-a.size:]


def _arb_advance(acc, input_deficit, delta, nphases, xlen):
    """Bookkeeping of one filt! call of FIRFilter{FIRArbitrary} with xlen >= inputDeficit samples
    (src/Filters/stream_filt.jl:567-625) in exact rational arithmetic: output j sits at total phase acc + j*delta and
    the loop `while xIdx <= xLen` keeps every j with inputDeficit + floor((acc + j*delta) / Nphi) <= xLen.
    Returns (number of outputs, inputDeficit after the call (:620), phiAccumulator after the call)."""
    A, Dl, N = Fraction(acc), Fraction(delta), nphases
    M = xlen - input_deficit + 1
    nout = math.ceil((M * N - A) / Dl)                           # number of j >= 0 with A + j*Dl < M*N
    P = A + nout * Dl                                            # phase after the last update! (:567-577)
    q = P // N
    new_acc = float(P - q * N)
    if new_acc >= N:                                             # rounding of a value just below Nphi
        new_acc = math.nextafter(float(N), 0.0)
    return nout, input_deficit + int(q) - xlen, new_acc


def filt_multirate(h, x, ratio, nphases=32):
    """filt(h::Vector, x::AbstractVector, ratio::Union{Integer,Rational}) and filt(h, x, rate::AbstractFloat, Nphi=32),
    src/Filters/stream_filt.jl:663-672."""
    return FIRFilter(h, ratio, nphases).filt(x)


def _arb_resample_call(sf, nx):
    """The filt! call that resample(x, rate::AbstractFloat) makes on each column (src/Filters/stream_filt.jl:696-725), as
    arguments of the arbitrary-rate kernel on the column itself.  sf is a fresh FIRArbitrary filter; undelay! (:706-714)
    is applied here.  The reference zero-pads the column to one sample more than inputlength(outLen, RoundUp) (:699) and
    filters [history; padded column]: the kernel sees the same samples when it reads min(nx, npad) samples of the column,
    zero elsewhere, with the newest sample of output 0 at index inputDeficit - 1.  The extra padding sample only
    guarantees that the exact count of outputs reaches outLen; the retained outputs never see it.
    Returns (outLen, samples read per column, n0, outputs the padded call would produce)."""
    outlen = math.ceil(nx * sf.rate)                                                          # :698
    sf.setphase(sf.timedelay())                                                               # undelay!
    npad = max(sf.inputlength(outlen, round_up=True), 0) + 1
    avail = 0
    if npad >= sf.input_deficit:                                                              # :590-594
        avail = _arb_advance(sf.phi_accumulator, sf.input_deficit, sf.delta, sf.nphases, npad)[0]
    return outlen, min(nx, npad), sf.input_deficit - 1, avail


def _resample_arbitrary(x, rate, h, nphases, dims):
    """resample(x, rate::AbstractFloat[, h, Nphi]; dims), src/Filters/stream_filt.jl:692-704, 751-775: a fresh FIRArbitrary
    filter per column, undelay!, zero-padding to inputlength(outLen, RoundUp), first ceil(length * rate) outputs.  Every
    column has the same phase state, so all columns go to the device in one launch.  A DeviceArray (a vector or a
    column-major len x nchan matrix resampled along dims=0) stays in device memory."""
    dev = isinstance(x, DeviceArray)
    if not dev:
        x = np.asarray(x)
    if not rate > 0.0:
        raise DomainError("rate must be greater than 0")
    sf = FIRFilter(h, rate, nphases)
    if dev:
        if x.ndim > 2 or (x.ndim == 2 and dims not in (None, 0)):
            raise ArgumentError("a DeviceArray is resampled as a vector or a len x nchan matrix along dims=0")
        nx = x.shape[0]
        ncols = x.shape[1] if x.ndim == 2 else 1
        outlen, m, n0, avail = _arb_resample_call(sf, nx)
        if ncols and avail < outlen:
            raise AssertionError("Resample output shorter than expected.")                   # :722
        plan = _lib.ResampleArbPlan(x.dtype, sf.h, sf.nphases)
        out = DeviceArray((outlen, ncols) if x.ndim == 2 else (outlen,), plan.out_dtype)
        plan.exec_batch_dev(x.ptr, m, nx, ncols, n0, sf.phi_accumulator, sf.delta, out.ptr, outlen, 0)
        from .device import sync
        sync()
        plan.close()
        return out
    if x.ndim > 1:
        if dims is None:
            raise ArgumentError("resample of an array needs `dims`")
        xm = np.moveaxis(x, dims, 0)
    else:
        xm = x
    nx = xm.shape[0]
    cols = xm.reshape(nx, -1)
    ncols = cols.shape[1]
    outlen, m, n0, avail = _arb_resample_call(sf, nx)
    if ncols == 0:
        res = np.empty((outlen, 0), dtype=np.float64)
    else:
        if avail < outlen:
            raise AssertionError("Resample output shorter than expected.")                   # :722
        xdt = _gpu_dtype(_promote(cols))
        plan = _lib.ResampleArbPlan(xdt, sf.h, sf.nphases)
        res = np.empty((outlen, ncols), dtype=plan.out_dtype, order="F")
        if x.ndim > 1:
            plan.exec_batch(np.asfortranarray(cols, dtype=xdt), m, nx, ncols, n0, sf.phi_accumulator, sf.delta, res, outlen)
        else:
            plan.exec(np.ascontiguousarray(cols[:m, 0], dtype=xdt), m, n0, sf.phi_accumulator, sf.delta, res[:, 0], outlen)
        plan.close()
    if x.ndim > 1:
        return np.moveaxis(res.reshape((outlen,) + xm.shape[1:]), 0, dims)
    return res.reshape(outlen)


def resample(x, rate, h=None, nphases=32, dims=None):
    """resample(x, rate[, h]; dims), src/Filters/stream_filt.jl:688-775: Integer / Rational rates through the rational
    polyphase kernel, floating-point rates through FIRArbitrary with `nphases` phases (default 32).
    Output eltype promote_type(eltype(h), eltype(x)) (:654); length ceil(length(x) * rate) (:698)."""
    if isinstance(rate, (float, np.floating)):
        return _resample_arbitrary(x, float(rate), h, int(nphases), dims)
    dev = isinstance(x, DeviceArray)
    if not dev:
        x = np.asarray(x)
    rate = _as_ratio(rate)
    if rate <= 0:
        raise ArgumentError("rate must be positive")
    if h is None:
        h = resample_filter(rate)
    h = np.asarray(h)
    if h.ndim != 1 or h.size == 0:
        raise ArgumentError("h must be a non-empty vector")
    if np.iscomplexobj(h):
        raise NotImplementedError("complex resampling taps are outside the GPU hot-path scope")
    hT = np.ascontiguousarray(h, dtype=np.float32 if h.dtype == np.float32 else np.float64)
    if dev:                                              # device pipeline form: a vector or a len x nchan matrix along dims=0
        if x.ndim > 2 or (x.ndim == 2 and dims not in (None, 0)):
            raise ArgumentError("a DeviceArray is resampled as a vector or a len x nchan matrix along dims=0")
        nout = math.ceil(x.shape[0] * rate)
        ncols = x.shape[1] if x.ndim == 2 else 1
        n0, phi0 = resample_phase(hT.size, rate)
        plan = _lib.ResamplePlan(x.dtype, hT, rate.numerator, rate.denominator)
        out = DeviceArray((nout, ncols) if x.ndim == 2 else (nout,), plan.out_dtype)
        plan.exec_dev(x.ptr, x.shape[0], ncols, n0, phi0, out.ptr, nout, 0)
        from .device import sync
        sync()
        plan.close()
        return out
    if x.ndim > 1:
        if dims is None:
            raise ArgumentError("resample of an array needs `dims`")
        xm = np.moveaxis(x, dims, 0)
    else:
        xm = x
    xdt = _gpu_dtype(_promote(xm))
    xF, nx, ncols = _cols(xm, xdt)
    nout = math.ceil(nx * rate)
    n0, phi0 = resample_phase(hT.size, rate)
    plan = _lib.ResamplePlan(xdt, hT, rate.numerator, rate.denominator)
    res = np.empty((nout, ncols), dtype=plan.out_dtype, order="F")
    plan.exec(xF, nx, ncols, n0, phi0, res, nout)
    plan.close()
    if x.ndim > 1:
        res = res.reshape((nout,) + xm.shape[1:])
        return np.moveaxis(res, 0, dims)
    return res.reshape(nout)
