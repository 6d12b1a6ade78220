"""Streaming multitaper spectrogram (MTSpectrogramStream; dspb200_stft_stream_exec(_dev) on a multitaper plan) and the
config forms of mt_spectrogram (MTSpectrogramConfig, mt_spectrogram(s, config), mt_spectrogram(s, mt_config, n_overlap),
mt_spectrogram_, allocate_output).

A stream call on a multitaper plan transforms the first kc complete segments of every channel's virtual column
[history; x] under every taper row of the plan and sums their PSD columns in taper order, so its columns equal
mt_spectrogram of the concatenated signal bit for bit.

CPU tests: the config's fields, times and refusals, allocate_output, and the stream front end against a stand-in library
(the calls it issues, residency, eltype and channel-shape rules, refused first calls, `out` checks).  GPU tests:
bit-identity with the one-shot mt_spectrogram for every fused size and eltype, taper sets (1, 2, 7 rows; dpss, custom and
eigenvalue-weighted), one- and two-sided, zero padding, overlaps, chunkings and channel counts, the Float32 1024-point warp
plan, the Float64 8192-point direct-load path and cuFFT sizes; host against device; the config forms against the keyword
form and the per-bin bound; launch counts; guard cells; the C ABI's refusals; caller streams and CUDA-graph capture; the
full-size 64-channel stream."""
import gc

import numpy as np
import pytest

import dspb200 as dsp
from dspb200 import _lib
from dspb200 import multitaper as mtm
from dspb200.device import DeviceArray
from dspb200.periodograms import stft_stream_step

import test_spectral_kernel_paths as kp
import test_stream_contract as sc
from test_spectral_kernel_paths import F32, F64, C64, C128, Guarded, same_bits
from test_stft_stream import _AddressOnly, _chunk_sizes, _signal

from oracle import periodograms as op


# =============================================================================== CPU: configs

class _StubMtPlan:
    """Stands in for the device plan: records its construction and the stream calls (nothing is launched)."""
    made, calls = [], []
    mt_spectrogram_batch_dev = None

    def __init__(self, dtype, n, noverlap, nfft, onesided, tapers):
        self.dtype, self.n, self.noverlap, self.nfft, self.onesided = np.dtype(dtype), n, noverlap, nfft, onesided
        self.tapers = np.array(tapers)
        self.nout = nfft // 2 + 1 if onesided else nfft
        _StubMtPlan.made.append(self)

    def stft_stream_dev(self, *args):
        _StubMtPlan.calls.append(("dev", self) + args)

    def stft_stream(self, *args):
        _StubMtPlan.calls.append(("host", self) + args)

    def mt_spectrogram_batch(self, s, length, nchan, out):
        _StubMtPlan.calls.append(("batch", self, s.dtype, length, nchan, out.shape))
        out[...] = 1

    def close(self):
        pass


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(mtm._lib, "MtPlan", _StubMtPlan)
    monkeypatch.setattr(dsp.periodograms, "DeviceArray", _AddressOnly)
    _StubMtPlan.made, _StubMtPlan.calls = [], []
    return _StubMtPlan


@pytest.mark.parametrize("n_samples,spw,nov,fs", [(10000, 1000, 500, 1), (10000, 1000, 0, 250.0), (999, 1000, 10, 1),
                                                  (1000, 1000, 999, 3.5), (4097, 256, 192, 8000.0)])
def test_config_fields_and_times(stub, n_samples, spw, nov, fs):
    cfg = dsp.MTSpectrogramConfig(n_samples, spw, nov, eltype=np.float32, fs=fs, nw=2)
    hop = spw - nov
    k = (n_samples - spw) // hop + 1 if n_samples >= spw else 0        # src/multitaper.jl:268-270
    assert cfg.n_samples == n_samples and cfg.n_overlap_samples == nov
    assert cfg.mt_config.n_samples == spw and cfg.mt_config.intype == F32 and cfg.mt_config.fs == fs
    assert np.array_equal(cfg.time, np.array([(spw / 2 + hop * i) / fs for i in range(k)]))
    # from an MTConfig: its fs, and the overlap's plan is built from the same pre-scaled rows
    mt = dsp.MTConfig(np.float64, spw, fs=fs, nw=2)
    cfg2 = dsp.MTSpectrogramConfig(n_samples, mt, nov)
    assert cfg2.mt_config is mt and np.array_equal(cfg2.time, cfg.time)
    p = mt.spectrogram_plan(nov)
    assert p.noverlap == nov and np.array_equal(p.tapers, mt.plan.tapers)
    assert mt.spectrogram_plan(nov) is p and mt.spectrogram_plan(0) is mt.plan
    nfft = 1 << (spw - 1).bit_length()                                 # the MTConfig default, nextpow(2, n)
    out = dsp.allocate_output(cfg)
    assert out.shape == (nfft // 2 + 1, k) and out.dtype == F32 and out.flags.f_contiguous
    out = dsp.allocate_output(dsp.MTSpectrogramConfig(n_samples, spw, nov, eltype=np.complex128, nw=2))
    assert out.shape == (nfft, k) and out.dtype == F64


def test_config_refusals(stub):
    with pytest.raises(dsp.ArgumentError):
        dsp.MTSpectrogramConfig(1000, 100, 100)                        # samples_per_window <= n_overlap
    with pytest.raises(dsp.ArgumentError):
        dsp.MTSpectrogramConfig(1000, 100, 150)
    mt = dsp.MTConfig(np.float32, 100, nfft=100, nw=2)
    with pytest.raises(dsp.ArgumentError):
        dsp.MTSpectrogramConfig(1000, mt, 100)
    with pytest.raises(dsp.ArgumentError):
        dsp.MTSpectrogramConfig(1000, mt, 50, nw=3)                    # an MTConfig or keyword settings
    with pytest.raises(dsp.DomainError):
        dsp.MTSpectrogramConfig(1000, mt, -1)
    with pytest.raises(dsp.ArgumentError):
        dsp.allocate_output(mt)
    cfg = dsp.MTSpectrogramConfig(1000, mt, 50)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_spectrogram(np.ones(1000, np.float32), cfg, 60)        # the config fixes the overlap
    # mt_spectrogram!: DimensionMismatch for the destination, then the signal (src/multitaper.jl:314-322)
    k = cfg.time.size
    with pytest.raises(dsp.DimensionMismatch):
        dsp.mt_spectrogram_(np.empty((51, k + 1), np.float32, order="F"), np.ones(1000, np.float32), cfg)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.mt_spectrogram_(np.empty((51, k), np.float32, order="F"), np.ones(1001, np.float32), cfg)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.mt_spectrogram_(np.empty((51, k), np.float32, order="F"), np.ones((1000, 2), np.float32), cfg)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_spectrogram_(np.empty((51, k), np.float64, order="F"), np.ones(1000, np.float32), cfg)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_spectrogram_(_AddressOnly((51, k), F32), np.ones(1000, np.float32), cfg)
    assert not [c for c in stub.calls if c[0] == "batch"]
    # accepted: a vector, a matrix, a C-ordered destination (filled through a column-major copy)
    out = np.zeros((51, k), np.float32)
    sp = dsp.mt_spectrogram_(out, np.ones(1000, np.float32), cfg)
    assert sp.power is out and np.all(out == 1) and np.array_equal(sp.time, cfg.time)
    assert stub.calls[-1][1] is mt.spectrogram_plan(50) and stub.calls[-1][2:] == (F32, 1000, 1, (51, k))
    sp = dsp.mt_spectrogram(np.ones((1000, 3), np.float32), mt, 50)
    assert sp.power.shape == (51, k, 3) and stub.calls[-1][2:] == (F32, 1000, 3, (51, k, 3))
    sp = dsp.mt_spectrogram(np.ones(1000, np.float32), mt)             # default overlap n >> 1
    assert sp.power.shape == (51, (1000 - 100) // 50 + 1) and stub.calls[-1][1].noverlap == 50


# =============================================================================== CPU: the stream front end

def test_stream_issues_psd_calls_with_unit_r(stub):
    n, nov = 256, 192
    hop = n - nov
    s = dsp.MTSpectrogramStream(n, nov, nw=2, ntapers=3, device=True)
    assert s.nfft == 256 and s.r == 1.0 and stub.made == []            # the MTConfig waits for the first chunk's eltype
    x = _AddressOnly((1000, 3), F32, _ptr=4096)
    sp = s.mt_spectrogram(x)
    kc, h = stft_stream_step(0, 1000, n, nov, True)
    (plan,) = stub.made
    assert plan.dtype == F32 and plan.noverlap == nov and plan.nfft == 256 and plan.onesided and plan.tapers.shape == (3, n)
    assert s.mt_config.plan is plan
    (call,) = stub.calls
    assert call[0] == "dev" and call[1] is plan
    hist_in, nhist, hist_out, ldh, xp, nx, nch, nseg, r, psd, outp, ldo = call[2:14]
    assert hist_in is None and nhist == 0 and ldh == n + hop - 1
    assert (xp, nx, nch, nseg, r, psd, outp, ldo) == (4096, 1000, 3, kc, 1.0, True, sp.power.ptr, kc)
    assert sp.power.shape == (129, kc, 3) and sp.power.dtype == F32
    assert np.array_equal(sp.time, (n / 2 + hop * np.arange(kc)) / 1) and sp.freq.size == 129
    assert s.history_len == h and s.nsegments == kc
    x2 = _AddressOnly((777, 3), F32)
    kc2, _ = stft_stream_step(h, 777, n, nov, True)
    sp2 = s.mt_spectrogram(x2)
    assert stub.calls[-1][2] == hist_out and stub.calls[-1][9] == kc2
    assert np.array_equal(sp2.time, (n / 2 + hop * np.arange(kc, kc + kc2)) / 1)
    held = s.history_len >= n
    g = s.nsegments
    f = s.finish()
    assert f.power.shape == (129, 1 if held else 0, 3) and np.array_equal(f.time, (n / 2 + hop * np.arange(g, g + held)))
    # complex chunks after reset(): a new MTConfig of that eltype, two-sided, ldh = n - 1
    s.reset()
    s.mt_spectrogram(_AddressOnly((700,), C64))
    assert stub.made[-1].dtype == C64 and not stub.made[-1].onesided and stub.calls[-1][5] == n - 1


def test_stream_from_an_mt_config(stub):
    mt = dsp.dpss_config(np.float64, 512, nw=3, ntapers=4, weight_by_evals=True, fs=100.0)
    s = dsp.MTSpectrogramStream(mt, device=False)
    assert s.noverlap == 256 and s.nfft == mt.nfft and s.fs == 100.0
    x = np.random.default_rng(0).standard_normal((3000, 2))
    sp = s.mt_spectrogram(x)
    call = stub.calls[-1]
    assert call[0] == "host" and call[1] is mt.spectrogram_plan(256) and call[1] is not mt.plan
    assert np.array_equal(call[1].tapers, mt.plan.tapers) and call[10] == 1.0 and call[11] is True
    assert sp.power.shape == (257, call[9], 2) and np.array_equal(sp.freq, mt.freq)
    assert np.array_equal(sp.time, (256 + 256 * np.arange(call[9])) / 100.0)
    with pytest.raises(dsp.ArgumentError):                             # the config fixes the eltype
        dsp.MTSpectrogramStream(mt).mt_spectrogram(x.astype(np.float32))
    with pytest.raises(dsp.ArgumentError):
        dsp.MTSpectrogramStream(dsp.MTConfig(np.complex64, 512, nw=3)).mt_spectrogram(np.ones(600, np.float32))


def test_stream_residency_eltype_shape_and_out_rules(stub):
    n = 256
    host = dsp.MTSpectrogramStream(n, nw=2)
    with pytest.raises(dsp.ArgumentError):
        host.mt_spectrogram(_AddressOnly((500, 3), F32))
    dev = dsp.MTSpectrogramStream(n, nw=2, device=True)
    with pytest.raises(dsp.ArgumentError):
        dev.mt_spectrogram(np.zeros((500, 3), F32))
    with pytest.raises(dsp.ArgumentError):
        dev.mt_spectrogram(_AddressOnly((500, 2, 2), F32))
    with pytest.raises(dsp.ArgumentError):                             # out too small: a refused first call
        dev.mt_spectrogram_(_AddressOnly((129, 0, 3), F32), _AddressOnly((1000, 3), F32))
    with pytest.raises(dsp.ArgumentError):                             # one-sided complex: the MTConfig refuses
        dsp.MTSpectrogramStream(n, onesided=True, device=True).mt_spectrogram(_AddressOnly((500,), C64))
    assert dev._key is None and stub.calls == []
    x = _AddressOnly((1000, 3), F32)
    dev.mt_spectrogram(x)
    for bad in (_AddressOnly((40, 3), F64), _AddressOnly((40, 4), F32), _AddressOnly((40,), F32)):
        with pytest.raises(dsp.ArgumentError):
            dev.mt_spectrogram(bad)
    hist_out = stub.calls[-1][4]
    x2 = _AddressOnly((600, 3), F32, _ptr=1 << 28)
    kc2, _ = stft_stream_step(dev.history_len, 600, n, n // 2, True)
    for out in (_AddressOnly((129, kc2 - 1, 3), F32), _AddressOnly((129, kc2, 3), F64), _AddressOnly((128, kc2, 3), F32),
                _AddressOnly((129, kc2, 2), F32), _AddressOnly((129, kc2, 3), F32, _ptr=(1 << 28) + 400),
                _AddressOnly((129, kc2, 3), F32, _ptr=hist_out + 8), np.zeros((129, kc2, 3), F32, order="F")):
        with pytest.raises(dsp.ArgumentError):
            dev.mt_spectrogram_(out, x2)
    with pytest.raises(dsp.ArgumentError):
        host.mt_spectrogram_(np.zeros((129, 10), F32), np.ones(2000, F32))     # not column-major
    assert len(stub.calls) == 1
    out = _AddressOnly((129, kc2 + 5, 3), F32)
    assert dev.mt_spectrogram_(out, x2) == kc2 and stub.calls[-1][12:14] == (out.ptr, kc2 + 5)


# =============================================================================== GPU helpers

def _config(dt, n, nfft, nov, kind, onesided=None):
    """An MTConfig for n-sample segments: 'dpss7' / 'dpss2' / 'dpss1' (nw 4, equal weights), 'custom' (two random rows of
    uneven energy), 'weighted' (dpss_config(weight_by_evals=True), three rows)."""
    if kind.startswith("dpss"):
        return dsp.MTConfig(dt, n, nfft=nfft, nw=4, ntapers=int(kind[4:]), onesided=onesided, noverlap=nov)
    if kind == "custom":
        rows = np.random.default_rng(n).standard_normal((n, 2)) * np.array([0.7, 1.9])
        return dsp.MTConfig(dt, n, nfft=nfft, window=rows, onesided=onesided, noverlap=nov)
    assert kind == "weighted"
    return dsp.dpss_config(dt, n, nw=2, ntapers=3, weight_by_evals=True, nfft=nfft, onesided=onesided, noverlap=nov)


def _oneshot(x, cfg, nov):
    """mt_spectrogram(column, cfg, nov) of each channel, one aligned device vector each: (nout, k, nchan)."""
    cols = [dsp.mt_spectrogram(dsp.to_device(np.ascontiguousarray(x[:, c])), cfg, nov).power.to_host() for c in range(x.shape[1])]
    return np.stack(cols, axis=2)


def _stream(x, sizes, cfg, nov, device=True):
    s = dsp.MTSpectrogramStream(cfg, nov, device=device)
    parts, a = [], 0
    for c in sizes:
        chunk = np.asfortranarray(x[a:a + c])
        a += c
        p = s.mt_spectrogram(dsp.to_device(chunk) if device else chunk).power
        parts.append(p.to_host() if device else p)
    f = s.finish().power
    parts.append(f.to_host() if device else f)
    return np.concatenate(parts, axis=1)


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and same_bits(a, b)


FUSED = [(dt, N) for dt in (F32, C64) for N in kp.SIZES] + [(dt, N) for dt in (F64, C128) for N in kp.SIZES if N <= 8192]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", FUSED, ids=[f"{d.name}-{N}" for d, N in FUSED])
def test_stream_is_bit_identical_every_fused_size(dt, N):
    rng = np.random.default_rng([N, dt.num])
    hop = N // 2
    for kind, ones in (("dpss7", None), ("custom", False if dt.kind == "f" else None), ("weighted", None)):
        cfg = _config(dt, N, N, N - hop, kind, ones)
        x = _signal(rng, (5 * N + 37, 3), dt)
        want = _oneshot(x, cfg, N - hop)
        for sizes in ([1 + 3 * hop // 2], [hop - 1], [hop], [hop + 1], [N - 1], [N], [N + hop], None):
            if sizes == [hop - 1] and N > 2048:
                continue                                          # thousands of launches: covered by the small sizes
            got = _stream(x, _chunk_sizes(rng, x.shape[0], sizes), cfg, N - hop)
            assert _same(got, want), (dt, N, kind, sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F64, C64, C128])
def test_overlaps_padding_tapers_and_channels(dt):
    rng = np.random.default_rng([12, dt.num])
    for n, nfft, kind in ((1024, 1024, "dpss1"), (1000, 1024, "dpss7"), (400, 512, "weighted"), (256, 256, "dpss2")):
        for nov in (0, n // 2, 3 * n // 4, n - 1):
            cfg = _config(dt, n, nfft, nov, kind)
            hop = n - nov
            nch = 70 if nov == n // 2 else 1 if nov == 0 else 3
            x = _signal(rng, (3 * n + 9 * hop + 5, nch), dt)
            want = _oneshot(x, cfg, nov)
            for sizes in ([hop + 1], [3, 5, 7], [1], None):
                if (hop == 1 and sizes not in ([3, 5, 7],)) or (sizes == [1] and x.shape[0] > 3000):
                    continue
                got = _stream(x, _chunk_sizes(rng, x.shape[0], sizes), cfg, nov)
                assert _same(got, want), (dt, n, nfft, kind, nov, sizes)


@pytest.mark.gpu
def test_float32_1024_warp_plan_against_the_aligned_one_shot_matrix():
    rng = np.random.default_rng(21)
    cfg = _config(F32, 1024, 1024, 768, "dpss7")
    x = _signal(rng, (40 * 256 + 768, 5), F32)                       # 16-byte aligned channels: the warp plan
    want = dsp.mt_spectrogram(dsp.to_device(x), cfg, 768).power.to_host()
    for sizes in ([4096], [1000, 3], None):
        assert _same(_stream(x, _chunk_sizes(rng, x.shape[0], sizes), cfg, 768), want), sizes
    # channels off 16-byte alignment: the one-shot matrix call runs the block kernel (test_mt_batched), the stream keeps the
    # warp plan -- the vector calls are the target
    xo = _signal(rng, (40 * 256 + 769, 3), F32)
    assert _same(_stream(xo, _chunk_sizes(rng, xo.shape[0], [3001]), cfg, 768), _oneshot(xo, cfg, 768))


@pytest.mark.gpu
def test_direct_load_path_float64_8192():
    rng = np.random.default_rng(3)
    cfg = _config(F64, 8192, 8192, 2048, "dpss2")
    x = _signal(rng, (6 * 8192 + 11, 1), F64)
    assert _same(_stream(x, _chunk_sizes(rng, x.shape[0], [5000, 8193, 1]), cfg, 2048), _oneshot(x, cfg, 2048))


def _cufft_launches(nt, nchan, kc, nfft, history):
    return nt * 3 * kp.cdiv(nchan * kc, kp.generic_batch(nfft)) + nt - 1 + (1 if history else 0) if kc else int(history)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,n,nfft", [(F32, 400, 400), (F32, 1000, 1000), (C64, 1000, 1000), (F64, 300, 320),
                                       (F32, 20000, 20000), (C128, 5000, 24000)])
def test_cufft_sizes(dt, n, nfft):
    rng = np.random.default_rng(n)
    nov = n // 4
    for kind in ("dpss7", "weighted"):
        cfg = _config(dt, n, nfft, nov, kind)
        x = _signal(rng, (7 * n + 13, 3), dt)
        want = _oneshot(x, cfg, nov)
        for sizes in ([n // 3], [n + 7], None):
            assert _same(_stream(x, _chunk_sizes(rng, x.shape[0], sizes), cfg, nov), want), (dt, n, nfft, kind, sizes)
    # launches: per taper three per batch of (channel, segment) pairs, an add per taper after the first, the history
    s = dsp.MTSpectrogramStream(cfg, nov, device=True)
    for c in (n - 1, 3 * n + 5, 40):
        h = s.history_len
        kc, newh = stft_stream_step(h, c, n, nov, not kp._cplx(dt))
        xd = dsp.to_device(_signal(rng, (c, 3), dt))
        before = dsp.launch_count()
        s.mt_spectrogram(xd)
        dsp.sync()
        assert dsp.launch_count() - before == _cufft_launches(cfg.ntapers, 3, kc, nfft, newh > 0), (c, kc)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", [(F32, 1024), (C64, 4096), (F32, 1000), (F64, 2048)])
def test_host_stream_equals_device_stream(dt, N):
    rng = np.random.default_rng(5)
    cfg = _config(dt, N, N, 3 * N // 4, "dpss7")
    x = _signal(rng, (6 * N + 3, 3), dt)
    hs, ds = dsp.MTSpectrogramStream(cfg, 3 * N // 4), dsp.MTSpectrogramStream(cfg, 3 * N // 4, device=True)
    a = 0
    for c in _chunk_sizes(rng, x.shape[0], None):
        chunk = np.asfortranarray(x[a:a + c])
        a += c
        assert _same(hs.mt_spectrogram(chunk).power, ds.mt_spectrogram(dsp.to_device(chunk)).power.to_host())
        assert hs.history_len == ds.history_len and hs.nsegments == ds.nsegments
        if hs.history is not None:
            assert _same(np.asfortranarray(hs.history), np.asfortranarray(ds.history.to_host()[:ds.history_len]))
    assert _same(hs.finish().power, ds.finish().power.to_host())


@pytest.mark.gpu
@pytest.mark.parametrize("dt,n,nfft", [(F32, 512, 512), (C64, 1024, 1024), (F32, 1000, 1000), (F64, 256, 300)])
def test_config_forms(dt, n, nfft):
    rng = np.random.default_rng([n, dt.num, 4])
    length, nov = 9 * n + 16, 3 * n // 4                               # 16-byte aligned channels: columns = vector calls
    x = np.asfortranarray(_signal(rng, (length, 3), dt))
    # where the parameters coincide, the config forms have the keyword form's bits (host and device)
    kw = dsp.mt_spectrogram(x, n, nov, nfft=nfft, nw=3, fs=2.0)
    mt = dsp.MTConfig(dt, n, nfft=nfft, nw=3, fs=2.0)                  # its `plan` has overlap 0: one more plan for nov
    cfg = dsp.MTSpectrogramConfig(length, mt, nov)
    for got in (dsp.mt_spectrogram(x, cfg), dsp.mt_spectrogram(x, mt, nov)):
        assert _same(got.power, kw.power) and np.array_equal(got.time, kw.time) and np.array_equal(got.freq, kw.freq)
    dx = dsp.to_device(x)
    assert _same(dsp.mt_spectrogram(dx, mt, nov).power.to_host(), kw.power)
    v = dsp.mt_spectrogram(np.ascontiguousarray(x[:, 1]), n, n // 2, nfft=nfft, nw=3)
    assert _same(dsp.mt_spectrogram(np.ascontiguousarray(x[:, 1]), dsp.MTConfig(dt, n, nfft=nfft, nw=3)).power, v.power)
    # mt_spectrogram! into preallocated destinations
    out = dsp.allocate_output(dsp.MTSpectrogramConfig(length, mt, nov))
    vec = np.ascontiguousarray(x[:, 2])
    assert dsp.mt_spectrogram_(out, vec, cfg).power is out and _same(out, kw.power[:, :, 2])
    outm = np.full(kw.power.shape, np.nan, dtype=kw.power.dtype, order="F")
    dsp.mt_spectrogram_(outm, x, cfg)
    assert _same(outm, kw.power)
    dout = DeviceArray(kw.power.shape, kw.power.dtype)
    assert dsp.mt_spectrogram_(dout, dx, cfg).power is dout and _same(dout.to_host(), kw.power)
    # eigenvalue-weighted tapers: every column within the per-bin bound of DESIGN.md section 4 (m = ntapers), and close to
    # the oracle's mt_pgram of its segment
    wc = dsp.dpss_config(dt, n, nw=3, weight_by_evals=True, nfft=nfft)
    sp = dsp.mt_spectrogram(x, wc, nov)
    rows, hop, nt = wc._rows, n - nov, wc.ntapers
    weights = wc.fs * np.sum(wc.window ** 2, axis=0) / wc.r
    b, mult = kp.bins_and_mult(nfft, wc.onesided)
    for c in range(3):
        for j in range(0, sp.time.size, 3):
            seg = x[j * hop:j * hop + n, c]
            refs = [kp.ref_segments(seg, n, n, nfft, rows[t]) for t in range(nt)]
            S = sum(np.abs(r[0][0, b]) ** 2 for r in refs)
            E = float(sum(r[1][0] for r in refs))
            kp.check_power(sp.power[:, j, c], S, E, mult, 1.0, kp.eps(dt), nfft, nt, ("weighted", c, j))
            o, _ = op.mt_pgram(seg, onesided=wc.onesided, nfft=nfft, window=wc.window, taper_weights=weights, f64=True)
            assert np.allclose(sp.power[:, j, c], o, rtol=0, atol=np.sqrt(kp.eps(dt)) * np.max(o))


@pytest.mark.gpu
def test_fused_launch_counts():
    rng = np.random.default_rng(9)
    for dt, n in ((F32, 1024), (F32, 512), (C64, 2048), (F64, 256)):
        s = dsp.MTSpectrogramStream(n, 3 * n // 4, nw=4, device=True)
        for c in (1, 700, n - 1, 3 * n + 5, 65536):
            x = dsp.to_device(_signal(rng, (c, 5), dt))
            before = dsp.launch_count()
            s.mt_spectrogram(x)
            assert dsp.launch_count() - before <= 2
        before = dsp.launch_count()
        s.mt_spectrogram(dsp.to_device(np.zeros((0, 5), dt, order="F")))
        assert dsp.launch_count() == before


@pytest.mark.gpu
@pytest.mark.parametrize("dt,nfft", [(F32, 1024), (C64, 512), (F32, 1000), (C128, 600)])
def test_guard_cells_and_c_abi_refusals(dt, nfft):
    """Calls on Guarded buffers: out and both histories keep every cell outside their range; psd_only = 0 or r != 1 on a
    multitaper plan is refused before any launch, in both forms."""
    rng = np.random.default_rng([nfft, dt.num, 6])
    n, nchan = nfft, 3
    hop = n // 4
    cfg = _config(dt, n, nfft, n - hop, "dpss2")
    plan = cfg.spectrogram_plan(n - hop)
    paired = not kp._cplx(dt)
    ldh = n - 1 + (hop if paired else 0)
    x = _signal(rng, (4 * n + 3 * hop + 1, nchan), dt)
    want = _oneshot(x, cfg, n - hop)
    re_ = kp._real(dt)
    gh = [Guarded(dt, ldh * nchan, rng), Guarded(dt, ldh * nchan, rng)]
    h, parts, a = 0, [], 0
    for c in (n + 5, 2 * hop + 1, x.shape[0] - n - 5 - 2 * hop - 1):
        kc, newh = stft_stream_step(h, c, n, n - hop, paired)
        gx = Guarded(dt, c * nchan, rng, np.asfortranarray(x[a:a + c]))
        go = Guarded(re_, plan.nout * (kc + 2) * nchan)
        before = dsp.launch_count()
        for bad in ((0, 1.0), (1, 2.0), (1, 0.5)):
            with pytest.raises(_lib.DSPB200Error):
                plan.stft_stream_dev(gh[0].ptr if h else None, h, gh[1].ptr, ldh, gx.ptr, c, nchan, kc, bad[1], bool(bad[0]),
                                     go.ptr, kc + 2, 0)
        assert dsp.launch_count() == before
        plan.stft_stream_dev(gh[0].ptr if h else None, h, gh[1].ptr, ldh, gx.ptr, c, nchan, kc, 1.0, True, go.ptr, kc + 2, 0)
        dsp.sync()
        o = go.data((plan.nout, kc + 2, nchan))                      # the ldo - kc columns past each channel's: NaN still
        assert np.isnan(o[:, kc:, :]).all()
        parts.append(o[:, :kc, :])
        gx.data()
        gh[0].data()
        gh = [gh[1], gh[0]]
        h, a = newh, a + c
    kc, _ = stft_stream_step(h, 0, n, n - hop, paired, final=True)
    go = Guarded(re_, plan.nout * max(kc, 1) * nchan)
    if kc:
        plan.stft_stream_dev(gh[0].ptr, h, gh[1].ptr, ldh, None, 0, nchan, kc, 1.0, True, go.ptr, kc, 0)
        dsp.sync()
        parts.append(go.data((plan.nout, kc, nchan)))
    gh[1].data()
    assert _same(np.concatenate(parts, axis=1), want)
    # the host form refuses the same calls before staging anything
    hx = np.asfortranarray(x[:n + 5])
    hout = np.zeros((plan.nout, 4, nchan), re_, order="F")
    hh = np.zeros((ldh, nchan), dt, order="F")
    before = dsp.launch_count()
    for psd, r in ((False, 1.0), (True, 3.0)):
        with pytest.raises(_lib.DSPB200Error):
            plan.stft_stream(None, 0, hh, ldh, hx, n + 5, nchan, 1, r, psd, hout, 4)
    assert dsp.launch_count() == before


# ---- caller streams and CUDA-graph capture: the harness of test_stream_contract.py on a multitaper plan

def _mt_stream_case(dt, nfft):
    def build(dsp_, scale):
        n, hop, _, _ = sc._spec_geometry(nfft, scale)
        tapers = sc._taps_rng(scale).standard_normal((3, n)) * 0.05
        plan = dsp_._lib.MtPlan(dt, n, n - hop, nfft, True, tapers)
        nhist, ldh, nx, nchan = n - hop, n, hop * 5 * scale + 3, 3
        nseg = (nhist + nx - n) // hop + 1
        return sc.Run([(dt, ldh * nchan), (dt, nx * nchan)], [(dt, ldh * nchan), (kp._real(dt), plan.nout * nseg * nchan)],
                      lambda i, o, st: plan.stft_stream_dev(i[0], nhist, o[0], ldh, i[1], nx, nchan, nseg, 1.0, True, o[1],
                                                            nseg, st), (plan,))
    return sc.Case(f"mt-stft_stream-{nfft}", ["dspb200_stft_stream_exec_dev"], "spectral/" + sc._spec_route(dt, nfft), build)


MT_CASES = [_mt_stream_case(F32, 1024), _mt_stream_case(F32, 1000)]


@pytest.fixture(scope="module")
def ctx():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("torch has no CUDA device")
    return sc.Ctx(dsp, torch)


@pytest.mark.gpu
@pytest.mark.parametrize("case", MT_CASES, ids=[c.name for c in MT_CASES])
def test_caller_stream_order_and_asynchrony(ctx, case):
    assert not case.sync
    sc.test_caller_stream_order_and_no_remembered_stream(dsp, ctx, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", MT_CASES, ids=[c.name for c in MT_CASES])
def test_cuda_graph_capture_and_replay(ctx, case):
    sc.test_cuda_graph_capture_and_replay(dsp, ctx, case)


@pytest.mark.gpu
def test_full_size_64_channels_in_65536_sample_blocks():
    rng = np.random.default_rng(4)
    nchan, length = 64, 1 << 22
    x = rng.standard_normal((length, nchan)).astype(F32, order="F")
    cfg = dsp.MTConfig(F32, 1024, nfft=1024, nw=4, noverlap=768)
    assert cfg.ntapers == 7
    dx = dsp.to_device(x)
    want = dsp.mt_spectrogram(dx, cfg, 768).power.to_host()           # one-shot matrix call (aligned: the warp plan)
    del dx
    s = dsp.MTSpectrogramStream(cfg, 768, device=True)
    parts = []
    for a in range(0, length, 65536):
        parts.append(s.mt_spectrogram(dsp.to_device(np.asfortranarray(x[a:a + 65536]))).power.to_host())
    parts.append(s.finish().power.to_host())
    assert _same(np.concatenate(parts, axis=1), want)
    gc.collect()
