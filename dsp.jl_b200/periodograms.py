"""periodogram / welch_pgram / spectrogram / stft front ends with the reference's signatures
(src/periodograms.jl), backed by libdspb200.  `welch_pgram!` is spelled `welch_pgram_`."""
import warnings

import numpy as np

from . import _lib
from .device import DeviceArray
from .errors import ArgumentError, DimensionMismatch, DomainError
from .util import fftabs2type, fftfreq, fftintype, fftouttype, nextfastfft, rfftfreq

_UNSET = object()


# --------------------------------------------------------------------------------------------- result types

class Periodogram:
    """Periodogram(power, freq), src/periodograms.jl:270-273."""

    def __init__(self, power, freq):
        self.power = power
        self.freq = freq


class Periodogram2:
    """Periodogram2(power, freq1, freq2), src/periodograms.jl:300-304: two-dimensional PSD; `freq` is the pair."""

    def __init__(self, power, freq1, freq2):
        self.power, self.freq1, self.freq2 = power, freq1, freq2

    @property
    def freq(self):
        return (self.freq1, self.freq2)


class Spectrogram:
    """Spectrogram(power, freq, time), src/periodograms.jl:773-777."""

    def __init__(self, power, freq, time):
        self.power = power
        self.freq = freq
        self.time = time


def power(p):
    """src/periodograms.jl:310."""
    return p.power


def freq(p):
    """src/periodograms.jl:329-333."""
    return p.freq


def time(p):
    """src/periodograms.jl:793."""
    return p.time


# --------------------------------------------------------------------------------------------- window / segmenting

def compute_window(window, n):
    """src/periodograms.jl:248-257 -> (window values as float64 or None, norm2)."""
    if window is None:
        return None, float(n)
    if callable(window):
        win = np.asarray(window(n), dtype=np.float64)
        return win, float(np.sum(win * win))
    win = np.asarray(window)
    if win.ndim != 1 or win.size != n:
        raise DimensionMismatch("length of window must match input")
    if np.iscomplexobj(win):
        raise NotImplementedError("complex windows are outside the GPU hot-path scope")
    return np.asarray(win, dtype=np.float64), float(np.sum(np.abs(win) ** 2))


def arraysplit_count(length, n, noverlap):
    """ArraySplit.k, src/periodograms.jl:49-50."""
    if not (0 <= noverlap < n):
        raise DomainError("noverlap must be between zero and n")     # :44
    return (length - n) // (n - noverlap) + 1 if length >= n else 0


def arraysplit(s, n, noverlap, nfft=None, window=None):
    """arraysplit(s, n, noverlap, nfft=n, window=nothing), src/periodograms.jl:134-137 (ArraySplit :32-73).
    Returns all k segments at once as a (k, nfft) array (`collect` of the reference's lazy iterator, :137):
    row i = [window .* s[i*hop : i*hop+n], zeros(nfft - n)], eltype fftintype(eltype(s))."""
    s = np.asarray(s)
    nfft = n if nfft is None else int(nfft)
    if not (0 <= noverlap < n):
        raise DomainError("noverlap must be between zero and n")     # :44
    if nfft < n:
        raise DomainError("nfft must be >= n")                      # :45
    sig = _signal(s)
    k = arraysplit_count(sig.size, n, noverlap)
    out = np.zeros((k, nfft), dtype=sig.dtype)
    if k == 0:
        return out
    win = None
    if window is not None:
        win = np.asarray(window)
        if win.size != n:
            raise DimensionMismatch("length of window must match input")
        win = np.asarray(win, dtype=np.float64)
    plan = _lib.SpecPlan(sig.dtype, n, noverlap, nfft, sig.dtype.kind != "c", win)
    plan.arraysplit(sig, out)
    plan.close()
    return out


def fftshift(p):
    """FFTW.fftshift(::Periodogram / ::Spectrogram), src/periodograms.jl:331-333, 778-780: two-sided spectra are
    rotated so frequencies ascend; one-sided ones are returned unchanged."""
    if isinstance(p, Periodogram2):                                                 # :336-337
        return Periodogram2(np.fft.fftshift(p.power), np.fft.fftshift(p.freq1), np.fft.fftshift(p.freq2))
    f = np.asarray(p.freq)
    if f.size == 0 or np.all(np.diff(f) > 0):
        return p
    if isinstance(p, Spectrogram):
        return Spectrogram(np.fft.fftshift(p.power, axes=0), np.fft.fftshift(f), p.time)
    return Periodogram(np.fft.fftshift(p.power), np.fft.fftshift(f))


def _signal(s):
    s = np.asarray(s)
    if s.ndim != 1:
        raise ArgumentError("expected a vector (the 2-D periodogram is outside the GPU hot-path scope)")
    return np.ascontiguousarray(s, dtype=fftintype(s.dtype))           # buffer eltype, :55


def _signal_matrix(s):
    """A len x nchan matrix of independent channels, column-major (one contiguous column per channel)."""
    return np.asfortranarray(s, dtype=fftintype(s.dtype))


# --------------------------------------------------------------------------------------------- WelchConfig

class WelchConfig:
    """WelchConfig(data_or_nsamples, eltype; n, noverlap, onesided, nfft, fs, window), src/periodograms.jl:516-587.
    Owns the device plan (segmenter + FFT + window), reusable across calls like the reference's plan/buffers.
    `data` may be a len x nchan matrix of channels: nsamples is then its number of rows."""

    def __init__(self, data, eltype=None, n=None, noverlap=None, onesided=None, nfft=None, fs=1, window=_UNSET):
        if eltype is None:
            data = np.asarray(data)
            nsamples, eltype = data.shape[0], data.dtype
        else:
            nsamples = int(data)
        eltype = np.dtype(eltype)
        n = nsamples >> 3 if n is None else int(n)
        noverlap = n >> 1 if noverlap is None else int(noverlap)
        cplx = eltype.kind == "c"
        onesided = (not cplx) if onesided is None else bool(onesided)
        nfft = nextfastfft(n) if nfft is None else int(nfft)
        if window is _UNSET:                                           # :582-587
            warnings.warn("Omitting `window` is deprecated; specify `window=None` for the old behaviour or "
                          "`window=hanning` for the future default.", DeprecationWarning, stacklevel=3)
            window = None
        if onesided and cplx:
            raise ArgumentError("cannot compute one-sided FFT of a complex signal")   # :564
        if nfft < n:
            raise DomainError("nfft must be >= n")                     # :565
        win, norm2 = compute_window(window, n)
        if not (0 <= noverlap < n):
            raise DomainError("noverlap must be between zero and n")   # ArraySplit :44
        self.nsamples, self.noverlap, self.onesided, self.nfft, self.fs = n, noverlap, onesided, nfft, fs
        self.window = win
        self.r = fs * norm2                                            # :568
        self.intype = fftintype(eltype)                                # eltype(inbuf) = float(T), :569
        self.freq = rfftfreq(nfft, fs) if onesided else fftfreq(nfft, fs)   # :573
        self.plan = _lib.SpecPlan(self.intype, n, noverlap, nfft, onesided, win)


def welch_pgram(s, n=None, noverlap=None, onesided=None, nfft=None, fs=1, window=_UNSET):
    """welch_pgram(s, n, noverlap; kw...) (src/periodograms.jl:647-649) or welch_pgram(s, config) (:702-705).
    A 2-D `s` (len x nchan) is the batched extension: every column is an independent signal, Welch-averaged with the same
    configuration in one launch; power is nout x nchan and the defaults come from len = size(s, 1)."""
    if isinstance(n, WelchConfig):
        config = n
    else:
        if isinstance(s, DeviceArray):
            nn = s.shape[0] >> 3 if n is None else int(n)
            config = WelchConfig(s.shape[0], s.dtype, n=nn, noverlap=(nn >> 1 if noverlap is None else noverlap),
                                 onesided=onesided, nfft=nfft, fs=fs, window=window)
        else:
            s = np.asarray(s)
            nn = s.shape[0] >> 3 if n is None else int(n)
            config = WelchConfig(s, n=nn, noverlap=(nn >> 1 if noverlap is None else noverlap), onesided=onesided,
                                 nfft=nfft, fs=fs, window=window)
    if isinstance(s, DeviceArray):
        return _welch_device(s, config)
    if np.ndim(s) == 2:
        sig = _signal_matrix(np.asarray(s))
        out = np.empty((config.freq.size, sig.shape[1]), dtype=fftabs2type(sig.dtype), order="F")
        return _welch_batch(out, sig, config)
    sig = _signal(s)
    out = np.empty(config.nfft // 2 + 1 if config.onesided else config.nfft, dtype=fftabs2type(sig.dtype))
    return _welch_helper(out, sig, config)


def filt_welch(x, n_or_b, b_or_config=None, config=None, nfft=None):
    """welch_pgram(filt(b, x), config) as one pipelined call: filt_welch(x, b, config) for a host array, or
    filt_welch(ptr, n, b, config) for a raw (ideally pinned) host pointer to `n` samples of eltype config.intype.
    The composition of the reference's `filt(b, x)` (src/dspbase.jl:14-15, FFT path src/Filters/filt.jl:445-521) and
    `welch_pgram(y, config)` (src/periodograms.jl:702-759); the stream is uploaded in chunks that overlap the kernels and
    the filter output never leaves the GPU (dspb200_filt_welch_exec).  Returns the Periodogram of the filtered stream."""
    if isinstance(x, (int, np.integer)):
        ptr_, n, b, cfg = int(x), int(n_or_b), b_or_config, config
        keep = None
    else:
        b, cfg = n_or_b, b_or_config
        keep = _signal(x)
        if keep.dtype != cfg.intype:
            raise ArgumentError(f"float(eltype(s)) = {keep.dtype} doesn't match the eltype of the input buffer: {cfg.intype}.")
        ptr_, n = _lib.ptr(keep), keep.size
    if not isinstance(cfg, WelchConfig):
        raise ArgumentError("filt_welch needs a WelchConfig")
    taps = np.ascontiguousarray(np.asarray(b), dtype=cfg.intype)
    if taps.ndim != 1 or taps.size == 0:
        raise ArgumentError("filter vector b must be non-empty")
    out = np.zeros(cfg.nfft // 2 + 1 if cfg.onesided else cfg.nfft, dtype=fftabs2type(cfg.intype))
    k = arraysplit_count(n, cfg.nsamples, cfg.noverlap)
    if k > 0:
        key = (taps.tobytes(), nfft)
        plans = cfg.__dict__.setdefault("_os_plans", {})
        osp = plans.get(key)
        if osp is None:
            osp = plans[key] = _lib.OsPlan(taps, 0 if nfft is None else int(nfft))
        cfg.plan.filt_welch_ptr(osp, ptr_, n, k * cfg.r, _lib.ptr(out))
    return Periodogram(out, cfg.freq)


def welch_pgram_(out, s, n=None, noverlap=None, onesided=None, nfft=None, fs=1, window=None):
    """welch_pgram!(out, s, config) (src/periodograms.jl:734-744) / welch_pgram!(out, s, n, noverlap; kw...) (:683-686).
    A 2-D `s` (len x nchan) needs an nout x nchan `out` (the batched extension of welch_pgram)."""
    if isinstance(n, WelchConfig):
        config = n
    else:
        s0 = np.asarray(s)
        nn = s0.shape[0] >> 3 if n is None else int(n)
        config = WelchConfig(s0, n=nn, noverlap=(nn >> 1 if noverlap is None else noverlap), onesided=onesided,
                             nfft=nfft, fs=fs, window=window)
    s = np.asarray(s)
    sdt = s.dtype
    if s.ndim == 2:
        if out.shape != (config.freq.size, s.shape[1]):
            raise DimensionMismatch(f"Expected `output` to be of size (length(config.freq), size(s, 2)) = "
                                    f"{(config.freq.size, s.shape[1])}; got {out.shape}")
    elif out.size != config.freq.size:
        raise DimensionMismatch(f"Expected `output` to be of length `length(config.freq)`; got {out.size} and {config.freq.size}")
    if out.dtype != fftabs2type(sdt):
        raise ArgumentError(f"Eltype of output ({out.dtype}) doesn't match the expected type: {fftabs2type(sdt)}.")
    if fftintype(sdt) != config.intype:
        raise ArgumentError(f"float(eltype(s)) = {sdt} doesn't match the eltype of the input buffer: {config.intype}.")
    if s.ndim == 2:
        return _welch_batch(out, _signal_matrix(s), config)
    return _welch_helper(out, _signal(s), config)


def _welch_helper(out, sig, config):
    """welch_pgram_helper!, src/periodograms.jl:746-759 (the segment loop runs on the GPU)."""
    if sig.dtype != config.intype:
        raise ArgumentError(f"float(eltype(s)) = {sig.dtype} doesn't match the eltype of the input buffer: {config.intype}.")
    k = arraysplit_count(sig.size, config.nsamples, config.noverlap)
    if k == 0:
        out[...] = 0
        return Periodogram(out, config.freq)
    r = k * config.r                                                   # :751
    res = out if out.flags.c_contiguous else np.empty(out.shape, dtype=out.dtype)
    config.plan.welch(sig, r, res)
    if res is not out:
        out[...] = res
    return Periodogram(out, config.freq)


def _welch_batch(out, sig, config):
    """welch_pgram_helper! on every column of a len x nchan matrix in one batched call; out is nout x nchan."""
    if sig.dtype != config.intype:
        raise ArgumentError(f"float(eltype(s)) = {sig.dtype} doesn't match the eltype of the input buffer: {config.intype}.")
    length, nchan = sig.shape
    k = arraysplit_count(length, config.nsamples, config.noverlap)
    if k == 0 or nchan == 0:
        out[...] = 0
        return Periodogram(out, config.freq)
    res = out if out.flags.f_contiguous else np.empty(out.shape, dtype=out.dtype, order="F")
    config.plan.welch_batch(sig, length, nchan, k * config.r, res)
    if res is not out:
        out[...] = res
    return Periodogram(out, config.freq)


def _welch_device(s, config):
    """welch_pgram on a device-resident vector or len x nchan matrix: only the power (nout, or nout x nchan) crosses PCIe."""
    if s.ndim not in (1, 2):
        raise ArgumentError("expected a vector or a len x nchan matrix")
    if s.dtype != config.intype:
        raise ArgumentError(f"float(eltype(s)) = {s.dtype} doesn't match the eltype of the input buffer: {config.intype}.")
    if s.ndim == 2:
        length, nchan = s.shape
        out = np.zeros((config.freq.size, nchan), dtype=fftabs2type(s.dtype), order="F")
        k = arraysplit_count(length, config.nsamples, config.noverlap)
        if k == 0 or nchan == 0:
            return Periodogram(out, config.freq)
        dout = DeviceArray(out.shape, out.dtype)
        config.plan.welch_batch_dev(s.ptr, length, nchan, k * config.r, dout.ptr, 0)
        dout.to_host(out)
        return Periodogram(out, config.freq)
    out = np.zeros(config.nfft // 2 + 1 if config.onesided else config.nfft, dtype=fftabs2type(s.dtype))
    k = arraysplit_count(s.shape[0], config.nsamples, config.noverlap)
    if k == 0:
        return Periodogram(out, config.freq)
    dout = DeviceArray(out.shape, out.dtype)
    config.plan.welch_dev(s.ptr, s.shape[0], k * config.r, dout.ptr, 0)
    dout.to_host(out)
    return Periodogram(out, config.freq)


def _periodogram2(s, nfft, fs, radialsum, radialavg):
    """periodogram(s::AbstractMatrix; nfft, fs, radialsum, radialavg), src/periodograms.jl:473-509."""
    if s.dtype.kind == "c":
        raise ArgumentError("the periodogram of a matrix takes a real signal")
    nfft = tuple(nextfastfft(n) for n in s.shape) if nfft is None else tuple(int(n) for n in nfft)
    if not (s.shape[0] <= nfft[0] and s.shape[1] <= nfft[1]):
        raise ArgumentError("nfft must be >= size(s)")
    if not (s.shape[0] > 1 and s.shape[1] > 1):
        raise ArgumentError("dimensions of s must be > 1")
    if radialsum and radialavg:
        raise ArgumentError("radialsum and radialavg are mutually exclusive")
    r = fs * s.size                                                                # fs * norm2, :491
    nmin = min(nfft)
    radial_freq = lambda n: np.arange(n, dtype=np.float64) * (fs / nmin)           # Frequencies(n, n, fs / nmin), :507
    ptype = 1 if radialsum else 2 if radialavg else 0
    if isinstance(s, DeviceArray):                                                 # device-resident matrix: result stays in HBM
        if s.dtype.kind != "f":
            raise ArgumentError("device matrices must be Float32 or Float64")
        T = fftabs2type(s.dtype)
        dout = DeviceArray(nfft if ptype == 0 else ((nmin >> 1) + 1,), T)
        _lib.periodogram2_dev(s.dtype, s.ptr, s.shape, nfft, r, ptype, dout.ptr)
        if ptype == 0:
            return Periodogram2(dout, fftfreq(nfft[0], fs), fftfreq(nfft[1], fs))
        return Periodogram(dout, radial_freq(dout.shape[0]))
    sig = np.asfortranarray(s, dtype=fftintype(s.dtype))
    T = fftabs2type(sig.dtype)
    if ptype == 0:
        out = np.empty(nfft, dtype=T, order="F")
        _lib.periodogram2(sig, nfft, r, 0, out)
        return Periodogram2(out, fftfreq(nfft[0], fs), fftfreq(nfft[1], fs))
    out = np.empty((nmin >> 1) + 1, dtype=T)
    _lib.periodogram2(sig, nfft, r, ptype, out)
    return Periodogram(out, radial_freq(out.size))


def periodogram(s, onesided=None, nfft=None, fs=1, window=None, radialsum=False, radialavg=False):
    """periodogram(s; onesided, nfft, fs, window), src/periodograms.jl:393-417: the single-segment case; a matrix gives
    the two-dimensional / radial periodogram (:473-509)."""
    if not isinstance(s, DeviceArray):
        s = np.asarray(s)
    if s.ndim == 2:
        return _periodogram2(s, nfft, fs, radialsum, radialavg)
    if s.ndim != 1:
        raise ArgumentError("expected a vector or a matrix")
    cplx = s.dtype.kind == "c"
    onesided = (not cplx) if onesided is None else bool(onesided)
    if onesided and cplx:
        raise ArgumentError("cannot compute one-sided FFT of a complex signal")      # :396
    nfft = nextfastfft(s.size) if nfft is None else int(nfft)
    if nfft < s.size:
        raise DomainError("nfft must be >= n = length(s)")                           # :397
    if s.size == 0:
        raise ArgumentError("empty signal")
    win, norm2 = compute_window(window, s.size)
    if isinstance(s, DeviceArray):                                                  # device-resident signal, small result to the host
        if s.dtype != fftintype(s.dtype):
            raise ArgumentError("device signals must be Float32, Float64, ComplexF32 or ComplexF64")
        plan = _lib.SpecPlan(s.dtype, s.size, 0, nfft, onesided, win)
        dout = DeviceArray((plan.nout,), fftabs2type(s.dtype))
        plan.welch_dev(s.ptr, s.size, fs * norm2, dout.ptr, 0)
        out = dout.to_host()
        plan.close()
        return Periodogram(out, rfftfreq(nfft, fs) if onesided else fftfreq(nfft, fs))
    sig = _signal(s)
    plan = _lib.SpecPlan(sig.dtype, s.size, 0, nfft, onesided, win)
    out = np.empty(plan.nout, dtype=fftabs2type(sig.dtype))
    plan.welch(sig, fs * norm2, out)
    plan.close()
    return Periodogram(out, rfftfreq(nfft, fs) if onesided else fftfreq(nfft, fs))


def stft(s, n=None, noverlap=None, psdonly=False, onesided=None, nfft=None, fs=1, window=None):
    """stft(s, n, noverlap[, PSDOnly()]; onesided, nfft, fs, window), src/periodograms.jl:872-897.
    A 2-D `s` (len x nchan) is the batched extension: returns nout x k x nchan."""
    dev = isinstance(s, DeviceArray)
    if not dev:
        s = np.asarray(s)
    batched = s.ndim == 2
    if s.ndim not in (1, 2):
        raise ArgumentError("expected a vector (or a len x nchan matrix for the batched form)")
    length = s.shape[0]
    cplx = s.dtype.kind == "c"
    n = length >> 3 if n is None else int(n)
    noverlap = n >> 1 if noverlap is None else int(noverlap)
    onesided = (not cplx) if onesided is None else bool(onesided)
    nfft = nextfastfft(n) if nfft is None else int(nfft)
    if onesided and cplx:
        raise ArgumentError("cannot compute one-sided FFT of a complex signal")      # :876
    win, norm2 = compute_window(window, n)
    k = arraysplit_count(length, n, noverlap)
    if nfft < n:
        raise DomainError("nfft must be >= n")                                        # ArraySplit :45
    dt = fftintype(s.dtype)
    nout = nfft // 2 + 1 if onesided else nfft
    odt = fftabs2type(dt) if psdonly else fftouttype(dt)
    if dev:                                              # device pipeline form: the spectrogram matrix stays in HBM
        nchan = s.shape[1] if batched else 1
        dout = DeviceArray((nout, k, nchan) if batched else (nout, k), odt)
        if k > 0 and nchan > 0:
            plan = _lib.SpecPlan(dt, n, noverlap, nfft, onesided, win)
            plan.stft_dev(s.ptr, length, nchan, fs * norm2, psdonly, dout.ptr, 0)
            from .device import sync
            sync()
            plan.close()
        return dout
    sig = np.asfortranarray(s.reshape(length, -1), dtype=dt)
    nchan = sig.shape[1]
    out = np.zeros((nout, k, nchan), dtype=odt, order="F")
    if k > 0 and nchan > 0:
        plan = _lib.SpecPlan(dt, n, noverlap, nfft, onesided, win)
        plan.stft(sig, length, nchan, fs * norm2, psdonly, out)
        plan.close()
    return out if batched else out[:, :, 0]


def spectrogram(s, n=None, noverlap=None, onesided=None, nfft=None, fs=1, window=None):
    """spectrogram(s, n, noverlap; onesided, nfft, fs, window), src/periodograms.jl:828-837.
    A 2-D `s` (len x nchan) is the batched extension: power is nout x k x nchan."""
    if not isinstance(s, DeviceArray):
        s = np.asarray(s)
    length = s.shape[0]
    cplx = s.dtype.kind == "c"
    n = length >> 3 if n is None else int(n)
    noverlap = n >> 1 if noverlap is None else int(noverlap)
    onesided = (not cplx) if onesided is None else bool(onesided)
    nfft = nextfastfft(n) if nfft is None else int(nfft)
    out = stft(s, n, noverlap, psdonly=True, onesided=onesided, nfft=nfft, fs=fs, window=window)
    k = out.shape[1]
    t = (n / 2 + (n - noverlap) * np.arange(k, dtype=np.float64)) / fs               # :835
    return Spectrogram(out, rfftfreq(nfft, fs) if onesided else fftfreq(nfft, fs), t)


# --------------------------------------------------------------------------------------------- streaming stft

def stft_stream_step(h, nx, n, noverlap, paired, final=False):
    """Bookkeeping of one STFTStream call, shared by the host and the device form: with h history samples and nx new
    ones, the call emits the first `kc` complete segments of the virtual column [history; x] and keeps v[kc*hop, h+nx) as
    the new history.  `paired` (real input): segments 2u and 2u+1 of the one-shot call share one complex FFT, so kc is
    even and a complete segment whose partner is not complete yet stays in the history -- except in the `final` call
    (finish()), which emits it unpaired.  Returns (kc, new h)."""
    k = arraysplit_count(h + nx, n, noverlap)
    kc = k - (k & 1) if paired and not final else k
    return kc, h + nx - kc * (n - noverlap)


class _ChunkStream:
    """What STFTStream and WelchStream share: the chunk checks (residency, eltype and channel shape fixed by the first chunk, a
    refused first call fixing nothing) and the pair of history buffers that every call reads one of and writes the other."""
    _a_name = ""

    def _check(self, x):
        name = type(self).__name__
        if self.device and not isinstance(x, DeviceArray):
            raise ArgumentError(f"a device {name} takes DeviceArrays (construct it without device=True for host arrays)")
        if not self.device and isinstance(x, DeviceArray):
            raise ArgumentError(f"a host {name} takes host arrays (construct it with device=True for DeviceArrays)")
        if self._finished:
            raise ArgumentError("the stream is finished: reset() starts a new one")
        if not self.device:
            x = np.asarray(x)
        if x.ndim not in (1, 2):
            raise ArgumentError(f"{self._a_name} chunk is a vector or a len x nchan matrix")
        dt = x.dtype if self.device else fftintype(x.dtype)
        if self.device and dt != fftintype(dt):
            raise ArgumentError("device chunks must be Float32, Float64, ComplexF32 or ComplexF64")
        key = (np.dtype(dt), tuple(x.shape[1:]))
        if self._key is None:
            self._setup(key[0], key[1])
        elif key != self._key:
            raise ArgumentError(f"this {name} streams {self._key[0]} chunks of channel shape {self._key[1]}; got "
                                f"{key[0]} {key[1]} (reset() starts a new stream)")
        if not self.device:
            x = np.asfortranarray(x, dtype=dt)
        return x

    def _nchan(self):
        return int(np.prod(self._key[1])) if self._key[1] else 1

    def _advance(self, launch, nx, nseg):
        """One library call with nx new samples and nseg segments -- launch(cur, nxt, h, nchan): history buffer cur (None: an
        empty history) in, nxt out -- then the swap of the history buffers and the new counts."""
        nchan = self._nchan()
        h = self.history_len
        newh = h + nx - nseg * self.hop
        if nchan and (nx or nseg):
            if self._hist is None:
                hshape = (self.ldh,) + self._key[1]
                self._hist = ([None, DeviceArray(hshape, self._key[0])] if self.device
                              else [None, np.zeros(hshape, dtype=self._key[0], order="F")])
            cur, nxt = self._hist
            launch(cur, nxt, h, nchan)
            if cur is None:                                 # the first call: an empty history in, none to reuse
                cur = (DeviceArray(nxt.shape, nxt.dtype) if self.device
                       else np.zeros(nxt.shape, dtype=nxt.dtype, order="F"))
            self._hist = [nxt, cur]
        self.history_len = newh
        if self._hist is not None:
            self.history = self._hist[0] if self.device else self._hist[0][:newh]
        self.nsegments += nseg

    def _chunk(self, x, *args):
        fresh = self._key is None
        x = self._check(x)
        try:
            return self._emit(x, *args)
        except ArgumentError:
            if fresh:                   # a refused first call leaves the stream as it was: no eltype or channel shape fixed
                self._key = None
            raise


class STFTStream(_ChunkStream):
    """stft / spectrogram of a signal that arrives in chunks (an extension: the reference's stft takes one vector).

    STFTStream(n, noverlap=n>>1, psdonly=False, onesided=None, nfft=nextfastfft(n), fs=1, window=None, device=False) takes
    the parameters of `stft`.  Every chunk `x` is a vector (nx,) or a column-major (nx, nchan) matrix of channels that share
    one sample count; `stft(x)` returns the columns the chunk completes -- (nout, kc) or (nout, kc, nchan) -- and for each
    channel they are exactly (bit for bit) the columns of stft(concatenation of all chunks so far) at the global segment
    indices nsegments .. nsegments + kc - 1.  For real input the one-shot call transforms segments 2u and 2u+1 as one complex
    FFT, so a real stream emits segments in those pairs only; `finish()` emits the held-back last segment, if any.  After
    finish(), further chunks raise ArgumentError until `reset()`.

    device=True: chunks and results are DeviceArrays; a chunk costs at most two kernel launches for power-of-two nfft (the
    cuFFT sizes take three per batch of segments plus one), no copy of the chunk and no host synchronisation.  `history` is
    then the current history buffer -- (ldh,) or (ldh, nchan), the first `history_len` rows valid.  A host stream takes host
    arrays (its `history` is the (history_len,) or (history_len, nchan) array).  A host stream refuses DeviceArrays and a
    device stream host arrays.  The first chunk fixes the eltype and channel shape; reset() drops them."""

    def __init__(self, n, noverlap=None, psdonly=False, onesided=None, nfft=None, fs=1, window=None, device=False):
        self.n = int(n)
        self.noverlap = self.n >> 1 if noverlap is None else int(noverlap)
        if not (0 <= self.noverlap < self.n):
            raise DomainError("noverlap must be between zero and n")                     # ArraySplit :44
        self.nfft = nextfastfft(self.n) if nfft is None else int(nfft)
        if self.nfft < self.n:
            raise DomainError("nfft must be >= n")                                        # ArraySplit :45
        self.hop = self.n - self.noverlap
        self.psdonly, self.fs, self.device = bool(psdonly), fs, bool(device)
        self._onesided_arg = onesided
        self.window, norm2 = compute_window(window, self.n)
        self.r = fs * norm2
        self._plans = {}
        self.reset()

    def reset(self):
        """Start a new stream: drops the history, the segment count, the eltype and the channel shape."""
        self.nsegments = 0
        self.history_len = 0
        self.history = None
        self._key = None             # (eltype, channel shape) fixed by the first chunk
        self._hist = None            # [current, next] history buffers
        self._finished = False
        return self

    # ---- first chunk: eltype, onesided, plan
    def _setup(self, dt, chan_shape):
        cplx = dt.kind == "c"
        onesided = (not cplx) if self._onesided_arg is None else bool(self._onesided_arg)
        if onesided and cplx:
            raise ArgumentError("cannot compute one-sided FFT of a complex signal")      # :876
        if dt not in self._plans:
            self._plans[dt] = _lib.SpecPlan(dt, self.n, self.noverlap, self.nfft, onesided, self.window)
        self.onesided, self.cplx = onesided, cplx
        self.nout = self.nfft // 2 + 1 if onesided else self.nfft
        self.odt = fftabs2type(dt) if self.psdonly else fftouttype(dt)
        # history capacity: n + hop - 1 samples for real input (a held-back segment), n - 1 for complex
        self.ldh = max(1, self.n - 1 + (0 if cplx else self.hop))
        self._key = (dt, chan_shape)

    _a_name = "an STFTStream"

    def _out_shape(self, cols):
        return (self.nout, cols) + self._key[1]

    def _run(self, x, nseg, out, ldo):
        """One library call on chunk x (nx may be 0): nseg segments into out (ldo columns per channel), then the swap of the
        history buffers."""
        nx = x.shape[0] if x is not None else 0
        plan = self._plans[self._key[0]]

        def launch(cur, nxt, h, nchan):
            if self.device:
                plan.stft_stream_dev(cur.ptr if cur is not None else None, h, nxt.ptr, self.ldh,
                                     x.ptr if x is not None else None, nx, nchan, nseg, self.r, self.psdonly,
                                     out.ptr if out is not None else None, ldo, 0)
            else:
                xx = x if x is not None else np.zeros((1,) + self._key[1], dtype=self._key[0], order="F")
                oo = out if out is not None else np.zeros(1, dtype=self.odt)
                plan.stft_stream(cur, h, nxt, self.ldh, xx, nx, nchan, nseg, self.r, self.psdonly, oo, ldo)
        self._advance(launch, nx, nseg)

    def _emit(self, x, out=None):
        kc, _ = stft_stream_step(self.history_len, x.shape[0], self.n, self.noverlap, not self.cplx)
        if out is None:
            out = (DeviceArray if self.device else (lambda s, d: np.zeros(s, dtype=d, order="F")))(self._out_shape(kc), self.odt)
            ldo = kc
        else:
            if self.device != isinstance(out, DeviceArray):
                raise ArgumentError("out must be a DeviceArray for a device STFTStream and a host array for a host one")
            if out.dtype != self.odt or out.ndim != 2 + len(self._key[1]) or out.shape[0] != self.nout or \
                    tuple(out.shape[2:]) != self._key[1]:
                raise ArgumentError(f"out must be a {self.odt} array of shape (nout = {self.nout}, >= {kc}) + {self._key[1]}")
            if out.shape[1] < kc:
                raise ArgumentError(f"out is too small: the chunk completes {kc} columns per channel, out holds {out.shape[1]}")
            if self.device:
                if out.overlaps(x) or (self._hist is not None and (out.overlaps(self._hist[0]) or out.overlaps(self._hist[1]))):
                    raise ArgumentError("out must not overlap the chunk or the stream's history")
            elif not out.flags.f_contiguous:
                raise ArgumentError("out must be Fortran-ordered (column-major)")
            ldo = out.shape[1]
        self._run(x if x.shape[0] else None, kc, out, ldo)
        return out, kc

    def stft(self, x):
        """The columns chunk x completes: (nout, kc) for a vector chunk, (nout, kc, nchan) for a matrix chunk."""
        return self._chunk(x)[0]

    def stft_(self, out, x):
        """stft(x) into `out`, whose second dimension holds at least kc columns; returns kc."""
        return self._chunk(x, out)[1]

    def spectrogram(self, x):
        """Spectrogram(power, freq, time) of the columns chunk x completes (psdonly streams): time of global segment g is
        (n/2 + g*hop)/fs, as in spectrogram (src/periodograms.jl:835)."""
        if not self.psdonly:
            raise ArgumentError("spectrogram() needs a psdonly STFTStream")
        g0 = self.nsegments
        p = self.stft(x)
        return Spectrogram(p, rfftfreq(self.nfft, self.fs) if self.onesided else fftfreq(self.nfft, self.fs),
                           self._times(g0, p.shape[1]))

    def _times(self, g0, kc):
        return (self.n / 2 + self.hop * np.arange(g0, g0 + kc, dtype=np.float64)) / self.fs

    def finish(self):
        """The held-back last segment of a real stream (0 or 1 column per channel, transformed unpaired as the one-shot call
        does when it has an odd number of segments); None before the first chunk.  Ends the stream until reset()."""
        if self._key is None:
            return None
        if self._finished:
            raise ArgumentError("the stream is finished: reset() starts a new one")
        kc, _ = stft_stream_step(self.history_len, 0, self.n, self.noverlap, not self.cplx, final=True)
        out = (DeviceArray if self.device else (lambda s, d: np.zeros(s, dtype=d, order="F")))(self._out_shape(kc), self.odt)
        if kc:
            self._run(None, kc, out, kc)
        self._finished = True
        return out


# --------------------------------------------------------------------------------------------- streaming welch_pgram

class WelchStream(_ChunkStream):
    """welch_pgram of a signal that arrives in chunks (an extension: the reference's welch_pgram takes one vector).

    WelchStream(n, noverlap=n>>1, onesided=None, nfft=nextfastfft(n), fs=1, window=None, device=False) takes the parameters
    and checks of WelchConfig.  Every chunk `x` is a vector (nx,) or a column-major (nx, nchan) matrix of channels that share
    one sample count; `update(x)` adds the power spectra of the segments the chunk completes -- every complete segment of
    the concatenation of all chunks so far, segment i starting at sample i*hop -- to a Float64 accumulator per channel and
    bin, and keeps the samples the next segment needs as the history (at most n - 1).  `welch_pgram()` can be read at any
    time and does not change the stream: it is welch_pgram of everything so far, r = nsegments*fs*norm2 (zeros before the
    first complete segment, as welch_pgram of a signal shorter than n).  One chunk from an empty history gives the power of
    welch_pgram of that chunk bit for bit for power-of-two nfft that have fused kernels; more chunks round differently, within
    the bound of DESIGN.md section 4.  The same chunks give the same bits.

    device=True: chunks and results are DeviceArrays and the accumulator stays in device memory; a chunk costs at most four
    kernel launches per group of channels for power-of-two nfft (one when it completes no segment), three per batch of
    segments plus one for cuFFT sizes, no copy of the chunk and no host synchronisation.  `history` is then the current
    history buffer -- (ldh,) or (ldh, nchan), the first `history_len` rows valid.  A host stream takes host arrays (its
    `history` is the (history_len,) or (history_len, nchan) array).  The first chunk fixes the eltype and channel shape;
    reset() drops them."""

    _a_name = "a WelchStream"

    def __init__(self, n, noverlap=None, onesided=None, nfft=None, fs=1, window=None, device=False):
        self.n = int(n)
        self.noverlap = self.n >> 1 if noverlap is None else int(noverlap)
        self.nfft = nextfastfft(self.n) if nfft is None else int(nfft)
        if self.nfft < self.n:
            raise DomainError("nfft must be >= n")                                        # :565
        self.window, norm2 = compute_window(window, self.n)
        if not (0 <= self.noverlap < self.n):
            raise DomainError("noverlap must be between zero and n")                     # ArraySplit :44
        self.hop = self.n - self.noverlap
        self.fs, self.device = fs, bool(device)
        self._onesided_arg = onesided
        self.r = fs * norm2                                                               # :568
        self._plans = {}
        self._finished = False
        self.reset()

    def reset(self):
        """Start a new stream: drops the history, the accumulated power, the segment count, the eltype and the channel shape."""
        self.nsegments = 0
        self.history_len = 0
        self.history = None
        self._key = None             # (eltype, channel shape) fixed by the first chunk
        self._hist = None            # [current, next] history buffers
        self._acc = None             # nout x nchan Float64 accumulator, written (not added to) by the first segment's call
        return self

    def _setup(self, dt, chan_shape):
        cplx = dt.kind == "c"
        onesided = (not cplx) if self._onesided_arg is None else bool(self._onesided_arg)
        if onesided and cplx:
            raise ArgumentError("cannot compute one-sided FFT of a complex signal")      # :564
        if dt not in self._plans:
            self._plans[dt] = _lib.SpecPlan(dt, self.n, self.noverlap, self.nfft, onesided, self.window)
        self.onesided, self.cplx = onesided, cplx
        self.nout = self.nfft // 2 + 1 if onesided else self.nfft
        self.odt = fftabs2type(dt)
        self.freq = rfftfreq(self.nfft, self.fs) if onesided else fftfreq(self.nfft, self.fs)   # :573
        self.ldh = max(1, self.n - 1)
        self._key = (dt, chan_shape)

    def _emit(self, x):
        nx = x.shape[0]
        kc, _ = stft_stream_step(self.history_len, nx, self.n, self.noverlap, False)
        plan = self._plans[self._key[0]]
        if self._acc is None:
            shape = (self.nout,) + self._key[1]
            self._acc = DeviceArray(shape, np.float64) if self.device else np.zeros(shape, dtype=np.float64, order="F")
        add = self.nsegments > 0                 # the first call that completes a segment writes the accumulator

        def launch(cur, nxt, h, nchan):
            if self.device:
                plan.welch_stream_dev(cur.ptr if cur is not None else None, h, nxt.ptr, self.ldh, x.ptr if nx else None, nx,
                                      nchan, kc, self._acc.ptr, add, 0)
            else:
                xx = x if nx else np.zeros((1,) + self._key[1], dtype=self._key[0], order="F")
                plan.welch_stream(cur, h, nxt, self.ldh, xx, nx, nchan, kc, self._acc, add)
        self._advance(launch, nx, kc)
        return kc

    def update(self, x):
        """Adds the segments chunk x completes to the accumulator; returns their number (per channel)."""
        return self._chunk(x)

    def welch_pgram(self):
        """Periodogram(power, freq) of everything streamed so far: power is (nout,) for vector chunks, (nout, nchan) for
        matrix chunks (a DeviceArray for a device stream)."""
        self._require_chunk()
        shape = (self.nout,) + self._key[1]
        out = DeviceArray(shape, self.odt) if self.device else np.empty(shape, dtype=self.odt, order="F")
        return self.welch_pgram_(out)

    def welch_pgram_(self, out):
        """welch_pgram() into `out` (shape (nout,) or (nout, nchan), the real eltype of the stream); returns the Periodogram."""
        self._require_chunk()
        shape = (self.nout,) + self._key[1]
        if self.device != isinstance(out, DeviceArray):
            raise ArgumentError("out must be a DeviceArray for a device WelchStream and a host array for a host one")
        if out.dtype != self.odt or tuple(out.shape) != shape:
            raise ArgumentError(f"out must be a {self.odt} array of shape {shape}")
        if self.device:
            if out.overlaps(self._acc):
                raise ArgumentError("out must not overlap the stream's accumulator")
        elif not out.flags.f_contiguous:
            raise ArgumentError("out must be Fortran-ordered (column-major)")
        nchan = self._nchan()
        plan = self._plans[self._key[0]]
        if self.nsegments == 0 or nchan == 0:                                  # fill!(out, 0), src/periodograms.jl:747
            if self.device:
                if out.nbytes:
                    out.copy_from_host(np.zeros(shape, dtype=self.odt, order="F"))
            else:
                out[...] = 0
        elif self.device:
            plan.welch_stream_power_dev(self._acc.ptr, nchan, self.nsegments * self.r, out.ptr, 0)
        else:
            plan.welch_stream_power(self._acc, nchan, self.nsegments * self.r, out)
        return Periodogram(out, self.freq)

    def _require_chunk(self):
        if self._key is None:
            raise ArgumentError("the WelchStream has had no chunk yet: its eltype and channel shape are not known")
