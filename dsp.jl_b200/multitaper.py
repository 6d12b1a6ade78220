"""Multitaper spectral estimation front ends (SURVEY.md 8f rank 1; reference src/multitaper.jl:5-790), backed by
libdspb200: `dpss`, `dpsseig`, `MTConfig`, `dpss_config`, `mt_pgram`, `MTSpectrogramConfig`, `mt_spectrogram`,
`mt_spectrogram_` (`mt_spectrogram!`), `allocate_output`, `MTSpectrogramStream`, `MTCrossSpectraConfig`, `MTCoherenceConfig`,
`mt_cross_power_spectra`, `mt_cross_power_spectra_` (`mt_cross_power_spectra!`), `mt_coherence`, `mt_coherence_`."""
import math

import numpy as np

from . import _lib
from .device import DeviceArray
from .errors import ArgumentError, DimensionMismatch, DomainError
from .periodograms import Periodogram, Spectrogram, STFTStream, arraysplit_count
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
        self._rows = (win / np.sqrt(self.r)[None, :]).T                              # rows pre-scaled by 1/sqrt(r_t)
        self.plan = _lib.MtPlan(self.intype, n_samples, noverlap, nfft, onesided, self._rows)
        self._spectrogram_plans = {int(noverlap): self.plan}

    def spectrogram_plan(self, n_overlap):
        """The plan of these taper rows with segments n_samples - n_overlap apart (a plan fixes its overlap): `plan` itself
        for the overlap it was built with, otherwise one more plan of the same rows, built on first use and kept."""
        n_overlap = int(n_overlap)
        plan = self._spectrogram_plans.get(n_overlap)
        if plan is None:
            plan = self._spectrogram_plans[n_overlap] = _lib.MtPlan(self.intype, self.n_samples, n_overlap, self.nfft,
                                                                     self.onesided, self._rows)
        return plan


def _mt_signal(s):
    """A vector or a len x nchan channel matrix (host array or DeviceArray): (s, device?, nchan or None for a vector)."""
    dev = isinstance(s, DeviceArray)
    if not dev:
        s = np.asarray(s)
    if s.ndim not in (1, 2):
        raise ArgumentError("expected a vector or a len x nchan matrix")
    return s, dev, (s.shape[1] if s.ndim == 2 else None)


def _mt_run(s, dev, nchan, config, shape, run, run_dev, out=None):
    """Run a multitaper plan over the columns of s (nchan None: a vector) into a result of `shape` + (nchan,): a new array,
    or `out` (checked by the caller: that shape and the real eltype of the config, a DeviceArray for a device signal)."""
    shape = shape + ((nchan,) if nchan is not None else ())
    nc = 1 if nchan is None else nchan
    odt = fftabs2type(config.intype)
    launch = all(shape)                                            # no channel or no segment: nothing to compute
    length = s.shape[0]
    if dev:                                                        # device-resident signal: the result stays in HBM
        if s.dtype != config.intype:
            raise ArgumentError(f"eltype of the device signal {s.dtype} does not match the config's {config.intype}")
        dout = DeviceArray(shape, odt) if out is None else out
        if launch:
            run_dev(s.ptr, length, nc, dout.ptr)
        return dout
    res = np.zeros(shape, dtype=odt, order="F") if out is None or not out.flags.f_contiguous else out
    if launch:
        run(np.asfortranarray(s.reshape(length, nc), dtype=config.intype), length, nc, res)
    if out is not None and res is not out:
        out[...] = res
    return res if out is None else out


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


class MTSpectrogramConfig:
    """MTSpectrogramConfig(n_samples, mt_config, n_overlap_samples) /
    MTSpectrogramConfig{T}(n_samples, samples_per_window, n_overlap_samples; fs, kwargs...), src/multitaper.jl:248-285:
    segments of mt_config.n_samples samples, n_overlap_samples apart, of a signal of n_samples; `time` holds the segment
    centres (samples_per_window/2 + hop*i)/fs.  Keyword settings (those of MTConfig) build the MTConfig of `eltype`."""

    def __init__(self, n_samples, mt_config_or_samples_per_window, n_overlap_samples, eltype=np.float64, fs=1, **kw):
        if isinstance(mt_config_or_samples_per_window, MTConfig):
            if kw:
                raise ArgumentError("pass either an MTConfig or keyword settings")
            mt = mt_config_or_samples_per_window
        else:
            mt = MTConfig(eltype, int(mt_config_or_samples_per_window), fs=fs, **kw)
        spw, n_overlap_samples = mt.n_samples, int(n_overlap_samples)
        if spw <= n_overlap_samples:
            raise ArgumentError("Need `samples_per_window > n_overlap_samples`; got `samples_per_window` = "
                                f"{spw} and `n_overlap_samples` = {n_overlap_samples}.")
        if n_overlap_samples < 0:
            raise DomainError("noverlap must be between zero and n")                  # ArraySplit, src/periodograms.jl:44
        hop = spw - n_overlap_samples
        k = arraysplit_count(int(n_samples), spw, n_overlap_samples)
        self.n_samples, self.n_overlap_samples, self.mt_config = int(n_samples), n_overlap_samples, mt
        self.time = (spw / 2 + hop * np.arange(k, dtype=np.float64)) / mt.fs


def _mt_spectrogram_config(s, config, out):
    """mt_spectrogram(s, config) / mt_spectrogram!(out, s, config) (out None: a new array), src/multitaper.jl:308-338."""
    s, dev, nchan = _mt_signal(s)
    mt = config.mt_config
    shape = (mt.freq.size, config.time.size)
    if out is not None:
        want = shape + ((nchan,) if nchan is not None else ())
        if tuple(out.shape) != want:
            raise DimensionMismatch(f"Expected `destination` to be of size `(length(config.mt_config.freq), "
                                    f"length(config.time))` = {want}; got {tuple(out.shape)}")
    if s.shape[0] != config.n_samples:
        raise DimensionMismatch(f"Expected `signal` to be of length `config.n_samples`; got {s.shape[0]} and "
                                f"{config.n_samples}")
    if out is not None:
        if dev != isinstance(out, DeviceArray):
            raise ArgumentError("the destination of a device signal is a DeviceArray, that of a host signal a host array")
        if out.dtype != fftabs2type(mt.intype):
            raise ArgumentError(f"Eltype of output ({out.dtype}) doesn't match the expected type: {fftabs2type(mt.intype)}.")
        if dev and out.overlaps(s):
            raise ArgumentError("the destination must not overlap the signal")
    plan = mt.spectrogram_plan(config.n_overlap_samples)
    power = _mt_run(s, dev, nchan, mt, (plan.nout, config.time.size), plan.mt_spectrogram_batch,
                    plan.mt_spectrogram_batch_dev, out)
    return Spectrogram(power, mt.freq, config.time)


def mt_spectrogram_(out, s, config):
    """mt_spectrogram!(destination, signal, config::MTSpectrogramConfig), src/multitaper.jl:308-324: the multitaper
    spectrogram into `out`, length(freq) x length(time) (x nchan for a len x nchan signal; a DeviceArray for a device
    signal, which may not overlap it).  Returns the Spectrogram, whose power is `out`."""
    if not isinstance(config, MTSpectrogramConfig):
        raise ArgumentError("mt_spectrogram_ takes an MTSpectrogramConfig")
    return _mt_spectrogram_config(s, config, out)


def mt_spectrogram(s, n=None, n_overlap=None, fs=1, onesided=None, nfft=None, nw=4, ntapers=None, window=None):
    """mt_spectrogram(signal, n, n_overlap; fs, onesided, kwargs...), src/multitaper.jl:262-404 (default nfft = nextpow(2, n)),
    mt_spectrogram(signal, config::MTSpectrogramConfig) and mt_spectrogram(signal, mt_config::MTConfig,
    n_overlap=mt_config.n_samples >> 1) (:330-391; the settings are then those of the config).
    A 2-D `s` (len x nchan) is the batched extension: power is nout x k x nchan, the layout of the batched spectrogram, and
    freq and time come from len = size(s, 1)."""
    if isinstance(n, MTSpectrogramConfig):
        if n_overlap is not None:
            raise ArgumentError("an MTSpectrogramConfig fixes the overlap")
        return _mt_spectrogram_config(s, n, None)
    if isinstance(n, MTConfig):
        s = _mt_signal(s)[0]
        config = MTSpectrogramConfig(s.shape[0], n, n.n_samples >> 1 if n_overlap is None else n_overlap)
        return _mt_spectrogram_config(s, config, None)
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


class MTSpectrogramStream(STFTStream):
    """mt_spectrogram of a signal that arrives in chunks (an extension: the reference's mt_spectrogram takes one vector).

    MTSpectrogramStream(mt_config, n_overlap=n>>1, device=False) streams with the tapers, weights, nfft, fs and sidedness of
    an MTConfig, whose eltype every chunk must have; MTSpectrogramStream(n, n_overlap=n>>1, fs=1, onesided=None,
    nfft=nextpow(2, n), nw=4, ntapers=None, window=None, taper_weights=None, device=False) builds the MTConfig from those
    settings and the first chunk's eltype.  It is a psdonly STFTStream whose plan holds the config's pre-scaled taper rows
    (r = 1): the chunk rules, `history`, `history_len`, `nsegments`, reset(), the pairing of real segments and the launch
    counts are those of STFTStream, and the columns a chunk completes are exactly (bit for bit) the columns of
    mt_spectrogram(concatenation of all chunks so far, mt_config, n_overlap) at the global segment indices.
    `mt_spectrogram(x)` returns their Spectrogram, `mt_spectrogram_(out, x)` writes them into `out` and returns their
    number, and `finish()` returns the Spectrogram of the held-back last segment of a real stream."""

    _a_name = "an MTSpectrogramStream"

    def __init__(self, config_or_n, n_overlap=None, fs=1, onesided=None, nfft=None, nw=4, ntapers=None, window=None,
                 taper_weights=None, device=False):
        self._given = config_or_n if isinstance(config_or_n, MTConfig) else None
        if self._given is not None:
            mt = self._given
            n, fs, nfft, onesided = mt.n_samples, mt.fs, mt.nfft, mt.onesided
        else:
            n = int(config_or_n)
            if n <= 0:
                raise ArgumentError("`n_samples` must be positive")
            nfft = (1 << (n - 1).bit_length()) if nfft is None else int(nfft)                   # nextpow(2, n)
            self._mt_kw = dict(fs=fs, nfft=nfft, window=window, nw=nw, ntapers=ntapers, taper_weights=taper_weights,
                               onesided=onesided)
        super().__init__(n, n_overlap, psdonly=True, onesided=onesided, nfft=nfft, fs=fs, device=device)
        self.r = 1.0                                        # the taper rows carry 1/sqrt(r_t)
        self._configs = {}
        self.mt_config = self._given

    def _setup(self, dt, chan_shape):
        mt = self._configs.get(dt)
        if mt is None:
            if self._given is not None:
                if dt != self._given.intype:
                    raise ArgumentError(f"this MTSpectrogramStream's MTConfig takes {self._given.intype} chunks; got {dt}")
                mt = self._given
            else:
                mt = MTConfig(dt, self.n, noverlap=self.noverlap, **self._mt_kw)
            self._configs[dt] = mt
            self._plans[dt] = mt.spectrogram_plan(self.noverlap)
        super()._setup(dt, chan_shape)
        self.mt_config = mt

    def _freq(self):
        return rfftfreq(self.nfft, self.fs) if self.onesided else fftfreq(self.nfft, self.fs)

    def mt_spectrogram(self, x):
        """Spectrogram(power, freq, time) of the columns chunk x completes: power is (nout, kc) for a vector chunk,
        (nout, kc, nchan) for a matrix chunk; the time of global segment g is (n/2 + g*hop)/fs."""
        return self.spectrogram(x)

    def mt_spectrogram_(self, out, x):
        """The columns chunk x completes into `out`, whose second dimension holds at least kc columns; returns kc."""
        return self.stft_(out, x)

    def finish(self):
        """Spectrogram of the held-back last segment of a real stream (0 or 1 column per channel); None before the first
        chunk.  Ends the stream until reset()."""
        g0 = self.nsegments
        p = super().finish()
        return None if p is None else Spectrogram(p, self._freq(), self._times(g0, p.shape[1]))


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


class MTCoherenceConfig:
    """MTCoherenceConfig(cs_config::MTCrossSpectraConfig) / MTCoherenceConfig(n_channels, n_samples_or_mt_config; eltype,
    fs, demean, freq_range, kwargs...), src/multitaper.jl:656-697: the coherence settings are those of the cross spectra
    config `cs_config` (built from the arguments of MTCrossSpectraConfig when none is given)."""

    def __init__(self, cs_config_or_n_channels, mt_config_or_n_samples=None, **kw):
        if isinstance(cs_config_or_n_channels, MTCrossSpectraConfig):
            if mt_config_or_n_samples is not None or kw:
                raise ArgumentError("pass either an MTCrossSpectraConfig or the arguments of one")
            self.cs_config = cs_config_or_n_channels
        else:
            self.cs_config = MTCrossSpectraConfig(cs_config_or_n_channels, mt_config_or_n_samples, **kw)

    @property
    def freq(self):
        return self.cs_config.freq


def allocate_output(config):
    """allocate_output(config), src/multitaper.jl:326-328, 506-511, 682-686: an uninitialised column-major array of the
    config's result: length(freq) x length(time) of the real eltype for an MTSpectrogramConfig, n_channels x n_channels x
    length(freq) of the complex eltype for an MTCrossSpectraConfig and of the real eltype for an MTCoherenceConfig."""
    if isinstance(config, MTSpectrogramConfig):
        mt = config.mt_config
        return np.empty((mt.freq.size, config.time.size), dtype=fftabs2type(mt.intype), order="F")
    if isinstance(config, (MTCrossSpectraConfig, MTCoherenceConfig)):
        cs = config if isinstance(config, MTCrossSpectraConfig) else config.cs_config
        t = fftouttype(cs.mt_config.intype) if isinstance(config, MTCrossSpectraConfig) else fftabs2type(cs.mt_config.intype)
        return np.empty((cs.n_channels, cs.n_channels, cs.nfreq), dtype=t, order="F")
    raise ArgumentError("allocate_output takes an MTSpectrogramConfig, an MTCrossSpectraConfig or an MTCoherenceConfig")


def _cross(signal, config, kw, coherence, out=None):
    """Cross spectra (coherence False) or coherence of an n_channels x n_samples matrix or, an extension, of the epoch mean
    of an n_channels x n_samples x n_epochs array (host or DeviceArray), into `out` (None: a new array; a DeviceArray for a
    device signal, which it may not overlap).  Returns (result, freq)."""
    dev = isinstance(signal, DeviceArray)
    if not dev:
        signal = np.asarray(signal)
    if signal.ndim not in (2, 3):
        raise ArgumentError("expected an n_channels x n_samples matrix or an n_channels x n_samples x n_epochs array")
    if isinstance(config, MTCoherenceConfig):
        config = config.cs_config
    if config is None:
        config = MTCrossSpectraConfig(signal.shape[0], signal.shape[1], eltype=signal.dtype, **kw)
    elif kw:
        raise ArgumentError("pass either a config or keyword settings")
    mt = config.mt_config
    if tuple(signal.shape[:2]) != (config.n_channels, mt.n_samples):
        raise DimensionMismatch("Size of `signal` does not match `(config.n_channels, config.mt_config.n_samples)`; got "
                                f"`size(signal)`={tuple(signal.shape)} but `(config.n_channels, config.mt_config.n_samples)`="
                                f"{(config.n_channels, mt.n_samples)}")
    shape = (config.n_channels, config.n_channels, config.nfreq)
    if out is not None and tuple(out.shape) != shape:
        raise DimensionMismatch(f"Size of `output` does not match `(config.n_channels, config.n_channels, "
                                f"length(config.freq_inds))`; got `size(output)`={tuple(out.shape)} but {shape}")
    nepochs = signal.shape[2] if signal.ndim == 3 else None
    if nepochs == 0:
        raise ArgumentError("n_epochs must be positive")
    if signal.dtype.kind == "c":
        raise ArgumentError("Only real data is supported (with the default choice of `onesided=true`) for this operation.")
    tout = fftabs2type(mt.intype) if coherence else fftouttype(mt.intype)
    if out is not None:
        if dev != isinstance(out, DeviceArray):
            raise ArgumentError("the destination of a device signal is a DeviceArray, that of a host signal a host array")
        if out.dtype != tout:
            raise ArgumentError(f"Eltype of output ({out.dtype}) doesn't match the expected type: {tout}.")
        if dev and out.overlaps(signal):
            raise ArgumentError("the destination must not overlap the signal")
    plan, args = mt.plan, (config.n_channels, config.demean, config.freq_lo, config.nfreq, coherence)
    if dev:                                                           # device-resident (column-major) array: result stays in HBM
        if signal.dtype != mt.intype:
            raise ArgumentError(f"eltype of the device signal {signal.dtype} does not match the config's {mt.intype}")
        dout = DeviceArray(shape, tout) if out is None else out
        if config.nfreq:
            if nepochs is None:
                plan.cross_spectra_dev(signal.ptr, *args, dout.ptr)
            else:
                plan.cross_spectra_epochs_dev(signal.ptr, args[0], nepochs, *args[1:], dout.ptr)
        return dout, config.freq
    sig = np.asfortranarray(signal, dtype=mt.intype)                  # the reference's layout: channel index fastest
    res = np.zeros(shape, dtype=tout, order="F") if out is None or not out.flags.f_contiguous else out
    if config.nfreq:
        if nepochs is None:
            plan.cross_spectra(sig, *args, res)
        else:
            plan.cross_spectra_epochs(sig, args[0], nepochs, *args[1:], res)
    if out is not None and res is not out:
        out[...] = res
    return (res if out is None else out), config.freq


def mt_cross_power_spectra(signal, config=None, **kw):
    """mt_cross_power_spectra(signal; fs, demean, freq_range, kwargs...) / (signal, config), src/multitaper.jl:518-640;
    signal is n_channels x n_samples.  An extension: an n_channels x n_samples x n_epochs signal gives the mean over the
    epochs of the cross spectra of its matrices signal[:, :, e] (demeaned per channel per epoch), summed in epoch order in
    the output eltype and divided by n_epochs part by part; one epoch gives the matrix result bit for bit."""
    return CrossPowerSpectra(*_cross(signal, config, kw, False))


def mt_cross_power_spectra_(out, signal, config=None, **kw):
    """mt_cross_power_spectra!(output, signal; kwargs...) / (output, signal, config), src/multitaper.jl:551-585: the cross
    spectra of a matrix or the epoch mean of a 3-D signal (see mt_cross_power_spectra) into `out`, n_channels x n_channels
    x length(config.freq) (a DeviceArray for a device signal).  Returns the CrossPowerSpectra, whose power is `out`."""
    if isinstance(config, MTCoherenceConfig):
        raise ArgumentError("mt_cross_power_spectra_ takes an MTCrossSpectraConfig")
    return CrossPowerSpectra(*_cross(signal, config, kw, False, out))


def mt_coherence(signal, config=None, **kw):
    """mt_coherence(signal; fs, demean, freq_range, kwargs...) / (signal, config), src/multitaper.jl:722-790; config is an
    MTCoherenceConfig or an MTCrossSpectraConfig.  A 3-D signal gives the coherence of the epoch-mean cross spectra."""
    return Coherence(*_cross(signal, config, kw, True))


def mt_coherence_(out, signal, config=None, **kw):
    """mt_coherence!(output, signal; kwargs...) / (output, signal, config::MTCoherenceConfig), src/multitaper.jl:756-778: the
    coherences of a matrix or of the epoch mean of a 3-D signal into `out`, n_channels x n_channels x length(freq) of the
    real eltype (a DeviceArray for a device signal).  Returns the Coherence, whose coherence is `out`."""
    if config is not None and not isinstance(config, MTCoherenceConfig):
        raise ArgumentError("mt_coherence_ takes an MTCoherenceConfig")
    return Coherence(*_cross(signal, config, kw, True, out))
