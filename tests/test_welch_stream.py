"""Streaming welch_pgram (WelchStream, dspb200_welch_stream_exec(_dev), dspb200_welch_stream_power(_dev)): chunked vectors
and len x nchan matrices.

A call adds the power spectra of every segment the chunk completes in every channel's virtual column [history; x] to a
Float64 accumulator and keeps the rest as the new history; the power is read at any time with welch_pgram's scaling.

CPU tests: the bookkeeping against arraysplit of the concatenation, and the argument, residency and accumulator rules with
a stand-in library.  GPU tests: one chunk from an empty history against the batched welch_pgram bit for bit for every fused
size and eltype (windows, one- and two-sided, n < nfft, unaligned, 1 / 3 / 70 channels, channel groups); many chunks
against a Float64 Welch of the concatenation within the per-bin bound of test_spectral_kernel_paths.py (restated below);
mid-stream reads; host against device; repeatability; guard cells around every buffer; launch counts; the C ABI's
refusals."""
import math

import numpy as np
import pytest

import dspb200 as dsp
from dspb200 import _lib
from dspb200.device import DeviceArray
from dspb200.periodograms import stft_stream_step
from oracle import periodograms as op

F32, F64, C64, C128 = (np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))


def _chunk_sizes(rng, total, sizes):
    """Consecutive chunk lengths covering `total` samples, cycling through `sizes` (None: random lengths, zeros included)."""
    out, a, i = [], 0, 0
    while a < total:
        c = int(rng.integers(0, 3 * 1024)) if sizes is None else sizes[i % len(sizes)]
        c = min(c, total - a)
        out.append(c)
        a, i = a + c, i + 1
    return out


# =============================================================================== CPU: bookkeeping

@pytest.mark.parametrize("n,noverlap", [(16, 0), (16, 8), (16, 12), (16, 15), (7, 3), (1, 0)])
def test_step_emits_every_complete_segment_of_the_concatenation(n, noverlap):
    rng = np.random.default_rng(n * 100 + noverlap)
    hop = n - noverlap
    for trial in range(40):
        h = emitted = seen = 0
        for nx in (int(v) for v in rng.integers(0, 3 * n + 2, int(rng.integers(1, 30)))):
            kc, newh = stft_stream_step(h, nx, n, noverlap, paired=False)
            seen += nx
            emitted += kc
            assert emitted == dsp.arraysplit_count(seen, n, noverlap)
            assert newh == seen - emitted * hop and 0 <= newh <= n - 1
            h = newh


# =============================================================================== CPU: argument rules with a stand-in library

class _FakePlan:
    calls = []

    def __init__(self, dtype, n, noverlap, nfft, onesided, window=None):
        self.dtype, self.n, self.noverlap, self.nfft, self.onesided = np.dtype(dtype), n, noverlap, nfft, onesided

    def welch_stream_dev(self, *args):
        _FakePlan.calls.append(("dev",) + args)

    def welch_stream(self, *args):
        _FakePlan.calls.append(("host",) + args)

    def welch_stream_power_dev(self, *args):
        _FakePlan.calls.append(("power_dev",) + args)

    def welch_stream_power(self, *args):
        _FakePlan.calls.append(("power",) + args)

    def close(self):
        pass


class _AddressOnly(DeviceArray):
    """A DeviceArray at a dummy address: nothing is allocated, read or launched.  New arrays get fresh addresses."""
    _next = [1 << 30]

    def __init__(self, shape, dtype, _base=None, _ptr=None):
        if _ptr is None:
            _ptr = _AddressOnly._next[0]
            _AddressOnly._next[0] += 1 << 24
        super().__init__(shape, dtype, _base=_base, _ptr=_ptr)


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(_lib, "SpecPlan", _FakePlan)
    monkeypatch.setattr(dsp.periodograms, "DeviceArray", _AddressOnly)
    _FakePlan.calls = []
    return _FakePlan


def test_parameter_checks_are_those_of_welchconfig(fake):
    with pytest.raises(dsp.DomainError):
        dsp.WelchStream(64, noverlap=64)
    with pytest.raises(dsp.DomainError):
        dsp.WelchStream(64, noverlap=-1)
    with pytest.raises(dsp.DomainError):
        dsp.WelchStream(64, nfft=32)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.WelchStream(64, window=np.ones(63))
    s = dsp.WelchStream(64, onesided=True, device=True)
    with pytest.raises(dsp.ArgumentError):
        s.update(_AddressOnly((100,), C64))
    assert s._key is None and fake.calls == []
    with pytest.raises(dsp.ArgumentError):
        s.welch_pgram()                                  # no chunk yet: no eltype or channel shape


def test_residency_eltype_and_channel_shape(fake):
    n, hop = 256, 128
    host = dsp.WelchStream(n)
    with pytest.raises(dsp.ArgumentError):
        host.update(_AddressOnly((500, 3), F32))
    dev = dsp.WelchStream(n, device=True)
    with pytest.raises(dsp.ArgumentError):
        dev.update(np.zeros((500, 3), F32))
    with pytest.raises(dsp.ArgumentError):
        dev.update(_AddressOnly((4, 2, 2), F32))
    assert fake.calls == [] and dev._key is None and host._key is None
    x = _AddressOnly((1000, 3), F32, _ptr=4096)
    kc, h = stft_stream_step(0, 1000, n, n - hop, False)
    assert dev.update(x) == kc == 6
    (call,) = fake.calls
    hist_in, nhist, hist_out, ldh, xp, nx, nch, nseg, accp, add = call[1:11]
    assert hist_in is None and nhist == 0 and ldh == n - 1
    assert (xp, nx, nch, nseg, add) == (4096, 1000, 3, kc, False)
    assert dev._acc.shape == (n // 2 + 1, 3) and dev._acc.dtype == F64 and accp == dev._acc.ptr
    assert dev.history_len == h and dev.nsegments == kc and dev.history.ptr == hist_out
    for bad in (_AddressOnly((40, 3), F64), _AddressOnly((40, 4), F32), _AddressOnly((40,), F32), np.zeros((40, 3), F32)):
        with pytest.raises(dsp.ArgumentError):
            dev.update(bad)
    assert len(fake.calls) == 1
    # later calls add, and swap the histories
    assert dev.update(_AddressOnly((300, 3), F32)) == stft_stream_step(h, 300, n, n - hop, False)[0]
    c2 = fake.calls[-1]
    assert c2[1] == hist_out and c2[2] == h and c2[9] == accp and c2[10] is True
    # the power: a (nout, 3) F32 DeviceArray, r = nsegments * fs * norm2
    p = dev.welch_pgram()
    assert isinstance(p.power, DeviceArray) and p.power.shape == (n // 2 + 1, 3) and p.power.dtype == F32
    assert fake.calls[-1][0] == "power_dev" and fake.calls[-1][1:4] == (accp, 3, dev.nsegments * n)
    assert np.array_equal(p.freq, dsp.rfftfreq(n, 1))
    for out in (_AddressOnly((n // 2 + 1, 3), F64), _AddressOnly((n // 2, 3), F32), np.zeros((n // 2 + 1, 3), F32),
                _AddressOnly((n // 2 + 1, 3), F32, _ptr=accp + 8)):
        with pytest.raises(dsp.ArgumentError):
            dev.welch_pgram_(out)
    # an empty chunk launches nothing
    ncalls = len(fake.calls)
    assert dev.update(_AddressOnly((0, 3), F32)) == 0 and len(fake.calls) == ncalls


def test_a_refused_first_call_fixes_nothing(fake):
    s = dsp.WelchStream(256, onesided=True, device=True)
    with pytest.raises(dsp.ArgumentError):
        s.update(_AddressOnly((1000, 3), C64))          # one-sided complex
    assert s._key is None and s._acc is None and fake.calls == []
    assert s.update(_AddressOnly((1000,), F64)) == 6
    assert s._key == (F64, ()) and s._acc.shape == (129,) and len(fake.calls) == 1


def test_accumulator_is_written_by_the_first_segment_and_after_reset(fake):
    n = 64
    s = dsp.WelchStream(n, window=dsp.hanning)
    x = np.zeros((n - 10, 2), F32, order="F")
    assert s.update(x) == 0                               # no segment yet: the call only keeps the history
    p = s.welch_pgram()
    assert p.power.shape == (n // 2 + 1, 2) and not p.power.any() and fake.calls[-1][0] == "host"
    assert fake.calls[-1][8] == 0 and fake.calls[-1][10] is False
    assert s.update(np.zeros((20, 2), F32)) == 1
    assert fake.calls[-1][8] == 1 and fake.calls[-1][10] is False        # the first segment writes acc
    assert s.update(np.zeros((40, 2), F32)) == 1 and fake.calls[-1][10] is True
    s.welch_pgram()
    norm2 = float(np.sum(dsp.hanning(n) ** 2))
    assert fake.calls[-1][0] == "power" and fake.calls[-1][2:4] == (2, 2 * norm2)
    s.reset()
    assert s.nsegments == 0 and s.history is None and s._key is None and s._acc is None
    assert s.update(np.zeros(3 * n, F64)) == 5 and fake.calls[-1][10] is False and s._acc.shape == (n // 2 + 1,)


# =============================================================================== GPU helpers

def _signal(rng, shape, dt):
    x = rng.standard_normal(shape)
    if dt.kind == "c":
        x = x + 1j * rng.standard_normal(shape)
    return np.asfortranarray(x.astype(dt))


def _same(a, b):
    """Bit for bit (a +0 / -0 or NaN payload difference counts)."""
    return (a.shape == b.shape and a.dtype == b.dtype and
            np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes())


def _stream(x, sizes, device=True, read_every=False, **kw):
    """x streamed in chunks of the given lengths; returns (power of everything, the stream, most segments of one call)."""
    s = dsp.WelchStream(device=device, **kw)
    a, most = 0, 0
    for c in sizes:
        chunk = np.asfortranarray(x[a:a + c])
        a += c
        most = max(most, s.update(dsp.to_device(chunk) if device else chunk))
        if read_every:
            s.welch_pgram()
    p = s.welch_pgram().power
    return (p.to_host() if device else p), s, most


C_FFT = 2.0


def power_bound(S, E, u, N, m):
    """test_spectral_kernel_paths.power_bound: an FFT accurate to c u log2(N) ||x|| per bin, squared, plus a register sum of
    m units."""
    cu = C_FFT * u * math.log2(N)
    return 2 * cu * np.sqrt(S * E) + cu * cu * E + m * u * S


def check_welch(P, x, n, noverlap, nfft, onesided, window, m, what=""):
    """P (nout, nchan) against a Float64 Welch of each column of x, bin by bin (test_spectral_kernel_paths.check_welch)."""
    dt = x.dtype
    u = float(np.finfo(F64 if dt in (F64, C128) else F32).eps)
    b = np.arange(nfft // 2 + 1) if onesided else np.arange(nfft)
    mult = np.ones(b.size)
    if onesided:
        mult[1:] = 2.0
        if nfft % 2 == 0:
            mult[-1] = 1.0
    win = None if window is None else window(n)
    norm2 = float(n) if win is None else float(np.sum(win * win))
    for c in range(x.shape[1]):
        segs = op.arraysplit(np.ascontiguousarray(x[:, c]), n, noverlap, nfft, win, f64=False).astype(np.complex128)
        X = np.fft.fft(segs, axis=1)
        S = np.mean(np.abs(X) ** 2, axis=0)[b]
        E = float(np.mean(np.sum(np.abs(segs) ** 2, axis=1)))
        err = np.abs(np.asarray(P[:, c], dtype=np.float64) * norm2 / mult - S)
        bad = np.flatnonzero(~(err <= power_bound(S, E, u, nfft, m)))
        assert bad.size == 0, (what, c, bad[:8])


def _oneshot(x, **kw):
    """The batched welch_pgram of the device matrix x (the comparison target of one-chunk streams)."""
    return dsp.welch_pgram(dsp.to_device(x), **kw).power


FUSED = [(F32, N) for N in (256, 512, 1024, 2048, 4096, 8192, 16384)] + [(F64, N) for N in (256, 512, 1024, 2048, 4096, 8192)] + \
        [(C64, N) for N in (256, 512, 1024, 2048, 4096, 8192, 16384)] + [(C128, N) for N in (256, 512, 1024, 2048, 4096, 8192)]


# =============================================================================== GPU: one chunk equals welch_pgram

@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", FUSED, ids=[f"{d.name}-{N}" for d, N in FUSED])
def test_one_chunk_is_bit_identical_to_batched_welch_pgram(dt, N):
    rng = np.random.default_rng(N)
    real = dt.kind == "f"
    cases = [dict(n=N, noverlap=N // 2, nfft=N, window=dsp.hanning),
             dict(n=N, noverlap=N // 4, nfft=N, window=None, onesided=False if real else None),
             dict(n=3 * N // 4, noverlap=N // 4, nfft=N, window=dsp.hamming)]
    for kw in cases:
        for nchan, length in ((1, 6 * N), (3, 5 * N + 37), (70, 2 * N + 1)):
            x = _signal(rng, (length, nchan), dt)
            want = _oneshot(x, **kw)
            got, s, _ = _stream(x, [length], **kw)
            assert _same(got, want), (dt, N, kw, nchan, length)
            assert s.nsegments == dsp.arraysplit_count(length, kw["n"], kw["noverlap"])


@pytest.mark.gpu
def test_one_chunk_in_channel_groups():
    # 32 MiB of Float32 16384-point partial rows hold 512 rows: 600 channels run in two groups (one chunk); a call with
    # seam units and interior units runs both transform launches per group, in groups of 256 (the second chunk)
    rng = np.random.default_rng(2)
    N, nchan = 16384, 600
    kw = dict(n=N, noverlap=N // 2, nfft=N, window=dsp.hanning)
    x = _signal(rng, (3 * N + 3, nchan), F32)
    assert _same(_stream(x, [x.shape[0]], **kw)[0], _oneshot(x, **kw))
    got, s, most = _stream(x, [N // 2 + 3, x.shape[0] - N // 2 - 3], **kw)
    assert most == 5 and s.nsegments == 5
    check_welch(got, x, N, N // 2, N, True, dsp.hanning, 3, "groups")


CUFFT_ONE = [(F32, 1000, 1000), (F64, 300, 320), (C128, 20000, 24000)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,n,nfft", CUFFT_ONE, ids=[f"{d.name}-{n}-{N}" for d, n, N in CUFFT_ONE])
def test_one_chunk_is_bit_identical_to_welch_pgram_at_cufft_sizes(dt, n, nfft):
    # one channel, more segments than one cuFFT batch: the stream and welch_pgram of the device vector (and of the one-column
    # matrix) run the same segment list through the same batches.  Not so for several channels: the stream packs the
    # channels' segments into shared batches.
    from test_spectral_kernel_paths import generic_batch
    rng = np.random.default_rng(nfft)
    hop = n - n // 2
    k = generic_batch(nfft) + 3
    length = (k - 1) * hop + n + 7
    x = _signal(rng, (length, 1), dt)
    for onesided in ((None, False) if dt.kind == "f" else (None,)):
        kw = dict(n=n, noverlap=n // 2, nfft=nfft, window=dsp.hanning, onesided=onesided)
        got, s, _ = _stream(x, [length], **kw)
        assert s.nsegments == k
        vec = dsp.welch_pgram(dsp.to_device(np.ascontiguousarray(x[:, 0])), **kw).power
        assert _same(got[:, 0], vec), (dt, n, nfft, onesided)
        assert _same(got, _oneshot(x, **kw)), (dt, n, nfft, onesided)


# =============================================================================== GPU: many chunks, within the bound

def _units(kc, dt):
    return kc if dt.kind == "c" else (kc + 1) // 2


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F64, C64, C128])
def test_chunkings_within_the_bound(dt):
    rng = np.random.default_rng(7)
    for n, noverlap, nfft in ((256, 128, 256), (512, 384, 512), (1000, 500, 1024), (4096, 2048, 4096), (256, 255, 256),
                              (512, 0, 512)):
        hop = n - noverlap
        kw = dict(n=n, noverlap=noverlap, nfft=nfft, window=dsp.hanning)
        x = _signal(rng, (3 * n + 7 * hop + 5, 3), dt)
        all_sizes = [[1 + 3 * hop // 2], [hop - 1], [hop], [hop + 1], [n - 1], [n], [n + hop], [3, 5, 7], [1001], None]
        for sizes in all_sizes:
            if sizes in ([hop - 1], [hop]) and hop < 4:
                continue                                          # hop = 1: the 1-sample chunks below
            if sizes == [1] or (sizes is not None and sizes[0] <= 8 and n > 512):
                continue
            got, s, most = _stream(x, _chunk_sizes(rng, x.shape[0], sizes), **kw)
            assert s.nsegments == dsp.arraysplit_count(x.shape[0], n, noverlap)
            check_welch(got, x, n, noverlap, nfft, dt.kind == "f", dsp.hanning, _units(most, dt), (dt, n, noverlap, sizes))
    # 1-sample chunks, hop = 1
    kw = dict(n=256, noverlap=255, nfft=256, window=dsp.hanning)
    x = _signal(rng, (300, 2), dt)
    got, _, most = _stream(x, [1] * 300, **kw)
    check_welch(got, x, 256, 255, 256, dt.kind == "f", dsp.hanning, _units(most, dt), (dt, "hop 1"))


@pytest.mark.gpu
@pytest.mark.parametrize("dt,n,nfft", [(F32, 1000, 1000), (C128, 20000, 24000), (F64, 300, 320)])
def test_cufft_sizes_within_the_bound(dt, n, nfft):
    rng = np.random.default_rng(n)
    for onesided in ((None, False) if dt.kind == "f" else (None,)):
        kw = dict(n=n, noverlap=n // 4, nfft=nfft, window=dsp.hanning, onesided=onesided)
        x = _signal(rng, (7 * n + 13, 3), dt)
        ones = dt.kind == "f" and onesided is None
        for sizes in ([n // 3], [n + 7], [x.shape[0]], None):
            got, _, most = _stream(x, _chunk_sizes(rng, x.shape[0], sizes), **kw)
            check_welch(got, x, n, n // 4, nfft, ones, dsp.hanning, max(1, most), (dt, n, sizes))


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", [(F32, 1024), (C64, 4096), (F32, 1000)])
def test_reading_mid_stream_gives_the_prefix_and_changes_nothing(dt, N):
    rng = np.random.default_rng(3)
    kw = dict(n=N, noverlap=N // 2, nfft=N, window=dsp.hanning)
    x = _signal(rng, (9 * N + 3, 3), dt)
    sizes = _chunk_sizes(rng, x.shape[0], [N + 17])
    s = dsp.WelchStream(device=True, **kw)
    a = 0
    for c in sizes:
        s.update(dsp.to_device(np.asfortranarray(x[a:a + c])))
        a += c
        p = s.welch_pgram().power.to_host()
        k = s.nsegments
        if k == 0:
            assert not p.any()
        else:
            check_welch(p, x[:(k - 1) * (N // 2) + N], N, N // 2, N, dt.kind == "f", dsp.hanning, k, (dt, a))
    quiet = _stream(x, sizes, **kw)[0]
    assert _same(quiet, _stream(x, sizes, read_every=True, **kw)[0])
    assert _same(quiet, _stream(x, sizes, **kw)[0])                   # repeatable


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", [(F32, 1024), (C64, 4096), (F32, 1000), (C128, 512)])
def test_host_stream_equals_device_stream(dt, N):
    rng = np.random.default_rng(5)
    kw = dict(n=N, noverlap=3 * N // 4, nfft=N, window=dsp.hanning)
    x = _signal(rng, (6 * N + 3, 3), dt)
    hs, ds = dsp.WelchStream(**kw), dsp.WelchStream(device=True, **kw)
    a = 0
    for c in _chunk_sizes(rng, x.shape[0], None):
        chunk = np.asfortranarray(x[a:a + c])
        a += c
        assert hs.update(chunk) == ds.update(dsp.to_device(chunk))
        assert hs.history_len == ds.history_len and hs.nsegments == ds.nsegments
        if hs._acc is not None and hs.nsegments:
            assert _same(hs._acc, ds._acc.to_host())
        if hs.history is not None:
            assert _same(np.asfortranarray(hs.history), np.asfortranarray(ds.history.to_host()[:ds.history_len]))
        assert _same(hs.welch_pgram().power, ds.welch_pgram().power.to_host())


GUARD, SENTINEL = 64, 1e6


class Guarded:
    """test_spectral_kernel_paths.Guarded: a device buffer of GUARD cells, `n` data cells and GUARD cells -- sentinels of
    magnitude 10^6 (input) or NaN (output) outside the data."""

    def __init__(self, dt, n, rng=None, data=None, offset=0):
        self.dt, self.n, self.lo = np.dtype(dt), n, GUARD + offset
        total = self.lo + n + GUARD
        if rng is None:
            host = np.full(total, np.nan, dtype=dt)
        else:
            s = rng.choice(np.array([-SENTINEL, SENTINEL]), total)
            if self.dt.kind == "c":
                s = s + 1j * rng.choice(np.array([-SENTINEL, SENTINEL]), total)
            host = s.astype(dt)
        if data is not None:
            host[self.lo:self.lo + n] = np.asarray(data).ravel(order="F")
        self.host = host
        self.buf = dsp.to_device(host)
        self.ptr = self.buf.ptr + self.lo * self.dt.itemsize

    def data(self, shape=None):
        h = self.buf.to_host()
        outside = np.concatenate([h[:self.lo], h[self.lo + self.n:]])
        want = np.concatenate([self.host[:self.lo], self.host[self.lo + self.n:]])
        assert np.array_equal(outside, want, equal_nan=True), "a cell outside the buffer's range changed"
        d = h[self.lo:self.lo + self.n]
        return d if shape is None else d.reshape(shape, order="F")


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", [(F32, 1024), (C64, 2048), (F64, 512), (F32, 1000)])
def test_guard_cells_around_every_buffer(dt, N):
    rng = np.random.default_rng(N)
    n, hop, nch = N, N // 2, 3
    plan = _lib.SpecPlan(dt, n, n - hop, N, dt.kind == "f", dsp.hanning(n))
    nout, ldh = plan.nout, n - 1
    x = _signal(rng, (4 * N + 5 * hop + 3, nch), dt)
    # the stream's calls by hand: chunks at odd offsets, histories in guarded buffers
    h, a, k = 0, 0, 0
    hist = Guarded(dt, ldh * nch, rng)
    acc = Guarded(F64, nout * nch)
    for c in (hop + 3, 2 * N + 1, x.shape[0] - 2 * N - hop - 4):
        kc, newh = stft_stream_step(h, c, n, n - hop, False)
        gx = Guarded(dt, c * nch, rng, np.asfortranarray(x[a:a + c]), offset=1)
        hout = Guarded(dt, ldh * nch, rng)
        plan.welch_stream_dev(hist.ptr if h else None, h, hout.ptr, ldh, gx.ptr, c, nch, kc, acc.ptr, k > 0, 0)
        dsp.sync()
        gx.data()
        hist.data()
        got_h = hout.data((ldh, nch))[:newh]
        v = x[a - h:a + c]
        assert _same(np.asfortranarray(got_h), np.asfortranarray(v[kc * hop:]))
        acc.data()
        hist, h, a, k = hout, newh, a + c, k + kc
    out = Guarded(F64 if dt in (F64, C128) else F32, nout * nch)
    plan.welch_stream_power_dev(acc.ptr, nch, k * float(np.sum(dsp.hanning(n) ** 2)), out.ptr, 0)
    dsp.sync()
    acc.data()
    check_welch(out.data((nout, nch)), x, n, n - hop, N, dt.kind == "f", dsp.hanning, k, (dt, N))


@pytest.mark.gpu
def test_launch_counts():
    rng = np.random.default_rng(9)
    for dt, n in ((F32, 1024), (F32, 512), (C64, 2048)):
        s = dsp.WelchStream(n, window=dsp.hanning, device=True)
        for c in (1, 700, n - 1, 3 * n + 5, 65536):
            x = dsp.to_device(_signal(rng, (c, 5), dt))
            h = s.history_len
            before = dsp.launch_count()
            kc = s.update(x)
            used = dsp.launch_count() - before
            assert used <= 4 and (kc > 0 or used == 1), (dt, n, c, h, kc, used)
        before = dsp.launch_count()
        s.update(dsp.to_device(np.zeros((0, 5), dt, order="F")))
        assert dsp.launch_count() == before
        s.welch_pgram()
        assert dsp.launch_count() == before + 1


@pytest.mark.gpu
def test_c_abi_refuses_bad_arguments_before_any_launch():
    n, hop, nch = 256, 128, 2
    plan = _lib.SpecPlan(F32, n, n - hop, n, True, None)
    ldh, nx, nseg, nout = n - 1, 1000, 6, n // 2 + 1
    hist_in, hist_out = DeviceArray((ldh, nch), F32), DeviceArray((ldh, nch), F32)
    x, acc, out = DeviceArray((nx, nch), F32), DeviceArray((nout, nch), F64), DeviceArray((nout, nch), F32)
    good = (hist_in.ptr, 0, hist_out.ptr, ldh, x.ptr, nx, nch, nseg, acc.ptr, False)
    before = dsp.launch_count()
    bad = [
        {2: hist_in.ptr},                                       # hist_out == hist_in
        {2: x.ptr},                                             # hist_out overlaps x
        {2: acc.ptr + 64},                                      # hist_out overlaps acc
        {8: x.ptr + 4},                                         # acc overlaps x
        {8: hist_in.ptr},                                       # acc overlaps hist_in
        {7: nseg + 2},                                          # segments past the virtual column
        {3: 100},                                               # the new history exceeds ldh
        {1: 10, 0: None},                                       # nhist > 0 without hist_in
        {5: -1},                                                # negative size
    ]
    for b in bad:
        args = list(good)
        for i, v in b.items():
            args[i] = v
        with pytest.raises(_lib.DSPB200Error):
            plan.welch_stream_dev(*args)
    with pytest.raises(_lib.DSPB200Error):
        _lib.check(_lib.lib.dspb200_welch_stream_exec_dev(plan.handle, *good[:9], 2, None))     # add not 0 / 1
    for args in ((acc.ptr, nch, 0.0, out.ptr), (acc.ptr, nch, 1.0, acc.ptr + 8), (acc.ptr, -1, 1.0, out.ptr)):
        with pytest.raises(_lib.DSPB200Error):
            plan.welch_stream_power_dev(*args)
    assert dsp.launch_count() == before
    plan.welch_stream_dev(*good)
    plan.welch_stream_power_dev(acc.ptr, nch, 6.0 * n, out.ptr)
    dsp.sync()
    assert 2 <= dsp.launch_count() - before <= 4
