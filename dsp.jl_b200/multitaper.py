"""Multitaper spectral estimation front ends (SURVEY.md 8f rank 1; reference src/multitaper.jl:5-790), backed by
libdspb200: `dpss`, `dpsseig`, `MTConfig`, `dpss_config`, `mt_pgram`, `mt_spectrogram`, `mt_cross_power_spectra`,
`mt_coherence`."""
import math

import numpy as np

from . import _lib
from .device import DeviceArray
from .errors import ArgumentError, DimensionMismatch, DomainError
from .periodograms import Periodogram, Spectrogram, arraysplit_count
from .util import fftabs2type, fftfreq, fftintype, fftouttype, nextfastfft, rfftfreq


def dpss(n, nw, ntapers=None):
    """dpss(n, nw, ntapers=ceil(2nw)-1), src/windows.jl:668-720: Slepian tapers as an (n, ntapers) matrix with unit-norm
    columns.  Restated as the reference computes them: the `ntapers` largest eigenpairs of the symmetric tridiagonal matrix
    (diagonal cospi(2nw/n) ((n-1)/2 - i)^2, off-diagonal i (n - i) / 2, :683-691) from LAPACK's tridiagonal eigensolver
    (Julia: eigen!(SymTridiagonal, range); here scipy.linalg.eigh_tridiagonal -- host-side taper design, not the hot loop),
    largest first; antisymmetric tapers start with a positive element (Slepian's convention, :697-707), symmetric ones are
    given a positive mean (what LAPACK returns there is not specified by the reference; MATLAB's dpss goldens have it so)."""
    from scipy.linalg import eigh_tridiagonal
    n = int(n)
    ntapers = math.ceil(2 * nw) - 1 if ntapers is None else int(ntapers)
    if not (0 < ntapers <= n):
        raise DomainError("ntapers must be in the interval (0, n]")
    if not (0 <= nw < n / 2):
        raise DomainError("nw must be in the interval [0, n/2)")
    i = np.arange(n, dtype=np.float64)
    dv = math.cos(2 * math.pi * nw / n) * ((n - 1) / 2 - i) ** 2
    ev = 0.5 * (i[1:] * n - i[1:] ** 2)
    if n == 1:
        return np.ones((1, 1))
    _, vec = eigh_tridiagonal(dv, ev, select="i", select_range=(n - ntapers, n - 1))
    rv = np.ascontiguousarray(vec[:, ::-1])                       # largest eigenvalue first
    for t in range(ntapers):
        col = rv[:, t]
        if t % 2 == 1:                                            # Julia's i = 2:2:size(rv, 2)
            nz = col[np.nonzero(col)[0][0]]
            if nz < 0:
                rv[:, t] = -col
        elif col.sum() < 0:
            rv[:, t] = -col
    return rv


class MTConfig:
    """MTConfig{T}(n_samples; fs, nfft, window, nw, ntapers, taper_weights, onesided), src/multitaper.jl:117-141."""

    def __init__(self, eltype, n_samples, fs=1, nfft=None, window=None, nw=4, ntapers=None, taper_weights=None,
                 onesided=None, noverlap=0):
        eltype = np.dtype(eltype)
        cplx = eltype.kind == "c"
        onesided = (not cplx) if onesided is None else bool(onesided)
        if onesided and cplx:
            raise ArgumentError("cannot compute one-sided FFT of a complex signal")
        if n_samples <= 0:
            raise ArgumentError("`n_samples` must be positive")
        nfft = (1 << (int(n_samples) - 1).bit_length()) if nfft is None else int(nfft)     # nextpow(2, n_samples)
        if nfft < n_samples:
            raise ArgumentError("Must have `nfft >= n_samples`")
        ntapers = math.ceil(2 * nw) - 1 if ntapers is None else int(ntapers)
        if window is None:
            win = dpss(n_samples, nw, ntapers)
            norm2 = np.ones(ntapers)
        else:
            win = np.asarray(window, dtype=np.float64)
            if win.ndim != 2 or win.shape[0] != n_samples:
                raise DimensionMismatch("window must be an n_samples x ntapers matrix")
            ntapers = win.shape[1]
            norm2 = np.sum(win * win, axis=0)
        w = np.full(ntapers, 1.0 / ntapers) if taper_weights is None else np.asarray(taper_weights, dtype=np.float64)
        self.n_samples, self.nfft, self.ntapers, self.fs, self.onesided = int(n_samples), nfft, ntapers, fs, onesided
        self.window = win
        self.r = fs * norm2 / w                                                      # :135-139
        self.freq = rfftfreq(nfft, fs) if onesided else fftfreq(nfft, fs)
        self.intype = fftintype(eltype)
        scaled = (win / np.sqrt(self.r)[None, :]).T                                  # rows pre-scaled by 1/sqrt(r_t)
        self.plan = _lib.MtPlan(self.intype, n_samples, noverlap, nfft, onesided, scaled)


def _mt_signal(s):
    """A vector or a len x nchan channel matrix (host array or DeviceArray): (s, device?, nchan or None for a vector)."""
    dev = isinstance(s, DeviceArray)
    if not dev:
        s = np.asarray(s)
    if s.ndim not in (1, 2):
        raise ArgumentError("expected a vector or a len x nchan matrix")
    return s, dev, (s.shape[1] if s.ndim == 2 else None)


def _mt_run(s, dev, nchan, config, shape, run, run_dev):
    """Run a multitaper plan over the columns of s (nchan None: a vector) into a result of `shape` + (nchan,)."""
    shape = shape + ((nchan,) if nchan is not None else ())
    nc = 1 if nchan is None else nchan
    odt = fftabs2type(config.intype)
    launch = all(shape)                                            # no channel or no segment: nothing to compute
    length = s.shape[0]
    if dev:                                                        # device-resident signal: the result stays in HBM
        if s.dtype != config.intype:
            raise ArgumentError(f"eltype of the device signal {s.dtype} does not match the config's {config.intype}")
        dout = DeviceArray(shape, odt)
        if launch:
            run_dev(s.ptr, length, nc, dout.ptr)
        return dout
    out = np.zeros(shape, dtype=odt, order="F")
    if launch:
        run(np.asfortranarray(s.reshape(length, nc), dtype=config.intype), length, nc, out)
    return out


def mt_pgram(s, config=None, onesided=None, nfft=None, fs=1, nw=4, ntapers=None, window=None):
    """mt_pgram(s; onesided, nfft=nextfastfft(length(s)), fs, nw, ntapers, window) / mt_pgram(s, config),
    src/multitaper.jl:178-242.  A 2-D `s` (len x nchan) is the batched extension: every column is estimated with the same
    configuration in one call, power is nout x nchan (a DeviceArray for device input) and the defaults come from
    len = size(s, 1)."""
    s, dev, nchan = _mt_signal(s)
    length = s.shape[0]
    if config is None:
        config = MTConfig(s.dtype, length, fs=fs, nfft=nextfastfft(length) if nfft is None else nfft, window=window, nw=nw,
                          ntapers=ntapers, onesided=onesided)
    if length != config.n_samples:
        raise DimensionMismatch("Expected `signal` to be of length `config.n_samples`")
    plan = config.plan
    power = _mt_run(s, dev, nchan, config, (plan.nout,), plan.mt_pgram_batch, plan.mt_pgram_batch_dev)
    return Periodogram(power, config.freq)


def mt_spectrogram(s, n=None, n_overlap=None, fs=1, onesided=None, nfft=None, nw=4, ntapers=None, window=None):
    """mt_spectrogram(signal, n, n_overlap; fs, onesided, kwargs...), src/multitaper.jl:262-404 (default nfft = nextpow(2, n)).
    A 2-D `s` (len x nchan) is the batched extension: power is nout x k x nchan, the layout of the batched spectrogram, and
    freq and time come from len = size(s, 1)."""
    s, dev, nchan = _mt_signal(s)
    length = s.shape[0]
    n = length >> 3 if n is None else int(n)
    n_overlap = n >> 1 if n_overlap is None else int(n_overlap)
    if n <= n_overlap:
        raise ArgumentError("Need `samples_per_window > n_overlap_samples`")
    config = MTConfig(s.dtype, n, fs=fs, nfft=nfft, window=window, nw=nw, ntapers=ntapers, onesided=onesided, noverlap=n_overlap)
    k = arraysplit_count(length, n, n_overlap)
    t = (n / 2 + (n - n_overlap) * np.arange(k, dtype=np.float64)) / fs
    plan = config.plan
    power = _mt_run(s, dev, nchan, config, (plan.nout, k), plan.mt_spectrogram_batch, plan.mt_spectrogram_batch_dev)
    return Spectrogram(power, config.freq, t)


def dpsseig(A, nw):
    """dpsseig(A, nw), src/windows.jl:739-775: concentration ratios (eigenvalues) of the tapers in the columns of A = dpss(..).
    Host-side design math like the window functions themselves."""
    A = np.asarray(A, dtype=np.float64)
    n = A.shape[0]
    if not (0 <= nw < n / 2):
        raise DomainError("nw must be in the interval [0, n/2)")
    w = nw / n
    seq = np.empty(n)
    seq[0] = 1.0
    seq[1:] = 2 * np.sinc(2 * w * np.arange(1, n))
    nfft = nextfastfft(2 * n - 1)
    spec = np.abs(np.fft.rfft(A, nfft, axis=0)) ** 2
    ac = np.fft.irfft(spec, nfft, axis=0)[:n] * nfft                 # brfft: unnormalised inverse
    return 2 * w * (seq @ ac) / nfft


def dpss_config(eltype, n_samples, nw=4, ntapers=None, fs=1, keep_only_large_evals=False, weight_by_evals=False, **kw):
    """dpss_config(T, n_samples; nw, ntapers, fs, keep_only_large_evals, weight_by_evals), src/multitaper.jl:52-77: an
    `MTConfig` whose tapers are optionally restricted to eigenvalues > 0.9 and weighted by their eigenvalues."""
    ntapers = int(2 * nw - 1) if ntapers is None else int(ntapers)
    window = dpss(n_samples, nw, ntapers)
    evals = None
    if keep_only_large_evals:
        evals = dpsseig(window, nw)
        keep = evals > 0.9
        window, evals = window[:, keep], evals[keep]
        ntapers = window.shape[1]
    if weight_by_evals:
        if evals is None:
            evals = dpsseig(window, nw)
        taper_weights = evals / evals.sum()
    else:
        taper_weights = np.full(ntapers, 1.0 / ntapers)
    return MTConfig(eltype, n_samples, window=window, nw=nw, ntapers=ntapers, taper_weights=taper_weights, fs=fs, **kw)


class CrossPowerSpectra:
    """CrossPowerSpectra(power, freq), src/multitaper.jl:398-405: power is n_channels x n_channels x length(freq)."""

    def __init__(self, power, freq):
        self.power, self.freq = power, freq


class Coherence:
    """Coherence(coherence, freq), src/multitaper.jl:703-719."""

    def __init__(self, coherence, freq):
        self.coherence, self.freq = coherence, freq


class MTCrossSpectraConfig:
    """MTCrossSpectraConfig{T}(n_channels, n_samples; fs, demean, freq_range, kwargs...) /
    MTCrossSpectraConfig(n_channels, mt_config; demean, freq_range), src/multitaper.jl:424-517."""

    def __init__(self, n_channels, mt_config_or_n_samples, eltype=np.float64, fs=1, demean=False, freq_range=None, **kw):
        if isinstance(mt_config_or_n_samples, MTConfig):
            mt = mt_config_or_n_samples
        else:
            mt = MTConfig(eltype, int(mt_config_or_n_samples), fs=fs, **kw)
        if mt.intype.kind == "c" or not mt.onesided:                                             # :411-416
            raise ArgumentError("Only real data is supported (with the default choice of `onesided=true`) for this operation.")
        self.n_channels, self.mt_config, self.demean, self.freq_range = int(n_channels), mt, bool(demean), freq_range
        if freq_range is not None:
            mask = (freq_range[0] < mt.freq) & (mt.freq < freq_range[-1])                        # :497-503
            idx = np.flatnonzero(mask)
        else:
            idx = np.arange(mt.freq.size)
        self.freq_lo = int(idx[0]) if idx.size else 0
        self.nfreq = int(idx.size)
        self.freq = mt.freq[idx]


def _cross(signal, config, kw, coherence):
    dev = isinstance(signal, DeviceArray)
    if not dev:
        signal = np.asarray(signal)
    if signal.ndim != 2:
        raise ArgumentError("expected an n_channels x n_samples matrix")
    if config is None:
        config = MTCrossSpectraConfig(signal.shape[0], signal.shape[1], eltype=signal.dtype, **kw)
    elif kw:
        raise ArgumentError("pass either a config or keyword settings")
    mt = config.mt_config
    if tuple(signal.shape) != (config.n_channels, mt.n_samples):
        raise DimensionMismatch("Size of `signal` does not match `(config.n_channels, config.mt_config.n_samples)`")
    if signal.dtype.kind == "c":
        raise ArgumentError("Only real data is supported (with the default choice of `onesided=true`) for this operation.")
    tout = fftabs2type(mt.intype) if coherence else fftouttype(mt.intype)
    if dev:                                                           # device-resident (column-major) matrix: result stays in HBM
        if signal.dtype != mt.intype:
            raise ArgumentError(f"eltype of the device signal {signal.dtype} does not match the config's {mt.intype}")
        dout = DeviceArray((config.n_channels, config.n_channels, config.nfreq), tout)
        if config.nfreq:
            mt.plan.cross_spectra_dev(signal.ptr, config.n_channels, config.demean, config.freq_lo, config.nfreq, coherence, dout.ptr)
        return dout, config.freq
    sig = np.asfortranarray(signal, dtype=mt.intype)                  # the reference's layout: channel index fastest
    out = np.zeros((config.n_channels, config.n_channels, config.nfreq), dtype=tout, order="F")
    if config.nfreq:
        mt.plan.cross_spectra(sig, config.n_channels, config.demean, config.freq_lo, config.nfreq, coherence, out)
    return out, config.freq


def mt_cross_power_spectra(signal, config=None, **kw):
    """mt_cross_power_spectra(signal; fs, demean, freq_range, kwargs...) / (signal, config), src/multitaper.jl:518-640;
    signal is n_channels x n_samples."""
    return CrossPowerSpectra(*_cross(signal, config, kw, False))


def mt_coherence(signal, config=None, **kw):
    """mt_coherence(signal; fs, demean, freq_range, kwargs...) / (signal, config), src/multitaper.jl:722-790."""
    return Coherence(*_cross(signal, config, kw, True))
