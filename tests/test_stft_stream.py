"""Streaming stft / spectrogram (STFTStream, dspb200_stft_stream_exec(_dev)): chunked vectors and len x nchan matrices.

A call transforms the first kc complete segments of every channel's virtual column [history; x] and keeps the rest as the
new history; a real stream emits segments in the pairs (2u, 2u+1) the one-shot call transforms together, so its columns
equal stft(concatenation) bit for bit.

CPU tests: the bookkeeping against arraysplit of the concatenation, and the argument, residency and overlap rules with a
stand-in library.  GPU tests: bit-identity with the one-shot stft of each channel for every dtype and fused size (the warp
plan of nfft = 1024 included), windows, PSD and raw, one- and two-sided, zero padding, overlaps, chunkings that put the
history at every alignment, the direct-load path, 1 / 3 / 70 channels, cuFFT sizes; host against device; the full-size
C4 stream; spectrogram times; launch counts; the C ABI's refusals."""
import numpy as np
import pytest

import dspb200 as dsp
from dspb200 import _lib
from dspb200.device import DeviceArray
from dspb200.periodograms import stft_stream_step

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
@pytest.mark.parametrize("paired", [True, False])
def test_step_matches_arraysplit_of_the_concatenation(n, noverlap, paired):
    rng = np.random.default_rng(n * 100 + noverlap)
    hop = n - noverlap
    for trial in range(40):
        sizes = [int(v) for v in rng.integers(0, 3 * n + 2, int(rng.integers(1, 30)))]
        h = emitted = seen = 0
        for nx in sizes:
            kc, newh = stft_stream_step(h, nx, n, noverlap, paired)
            seen += nx
            assert kc >= 0 and (kc % 2 == 0 or not paired)
            assert newh == h + nx - kc * hop and 0 <= newh <= (n + hop - 1 if paired else n - 1)
            # the emitted segments are the first ones of the concatenation, and all complete ones but a held-back partner
            total = dsp.arraysplit_count(seen, n, noverlap)
            assert emitted + kc <= total and total - (emitted + kc) <= (1 if paired else 0)
            # the new history starts at the next segment's first sample
            assert newh == seen - (emitted + kc) * hop
            h, emitted = newh, emitted + kc
        # finish(): the held-back segment
        kf, hf = stft_stream_step(h, 0, n, noverlap, paired, final=True)
        assert kf == (1 if paired and h >= n else 0) and hf == h - kf * hop
        assert emitted + kf == dsp.arraysplit_count(seen, n, noverlap)


# =============================================================================== CPU: argument rules with a stand-in library

class _FakePlan:
    calls = []

    def __init__(self, dtype, n, noverlap, nfft, onesided, window=None):
        self.dtype, self.n, self.noverlap, self.nfft, self.onesided = np.dtype(dtype), n, noverlap, nfft, onesided

    def stft_stream_dev(self, *args):
        _FakePlan.calls.append(("dev",) + args)

    def stft_stream(self, *args):
        _FakePlan.calls.append(("host",) + args)

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


def test_parameter_checks_are_those_of_stft(fake):
    with pytest.raises(dsp.DomainError):
        dsp.STFTStream(64, noverlap=64)
    with pytest.raises(dsp.DomainError):
        dsp.STFTStream(64, noverlap=-1)
    with pytest.raises(dsp.DomainError):
        dsp.STFTStream(64, nfft=32)
    s = dsp.STFTStream(64, onesided=True, device=True)
    with pytest.raises(dsp.ArgumentError):
        s.stft(_AddressOnly((100,), C64))
    assert fake.calls == []


def test_a_refused_first_call_fixes_nothing(fake):
    s = dsp.STFTStream(256, psdonly=True, device=True)
    with pytest.raises(dsp.ArgumentError):
        s.stft_(_AddressOnly((129, 0, 3), F32), _AddressOnly((1000, 3), F32))      # out too small
    assert s._key is None and fake.calls == []
    y = s.stft(_AddressOnly((1000,), F64))                                          # another eltype and channel shape
    assert y.dtype == F64 and y.ndim == 2 and len(fake.calls) == 1


def test_residency_and_argument_rules_fail_before_any_launch(fake):
    n, hop = 256, 128
    host = dsp.STFTStream(n, psdonly=True)
    with pytest.raises(dsp.ArgumentError):
        host.stft(_AddressOnly((500, 3), F32))
    dev = dsp.STFTStream(n, psdonly=True, device=True)
    with pytest.raises(dsp.ArgumentError):
        dev.stft(np.zeros((500, 3), F32))
    with pytest.raises(dsp.ArgumentError):
        dev.stft(_AddressOnly((4, 2, 2), F32))
    with pytest.raises(dsp.ArgumentError):
        dsp.STFTStream(n, device=True).spectrogram(_AddressOnly((500,), F32))        # not a psdonly stream
    assert fake.calls == [] and dev._key is None
    x = _AddressOnly((1000, 3), F32, _ptr=4096)
    y = dev.stft(x)                                      # segments 0..5 complete, 0..5 emitted (even)
    kc, h = stft_stream_step(0, 1000, n, n - hop, True)
    assert isinstance(y, DeviceArray) and y.shape == (n // 2 + 1, kc, 3) and y.dtype == F32
    (call,) = fake.calls
    hist_in, nhist, hist_out, ldh, xp, nx, nch, nseg, r, psd, outp, ldo = call[1:13]
    assert hist_in is None and nhist == 0 and ldh == n + hop - 1
    assert (xp, nx, nch, nseg, psd, outp, ldo) == (4096, 1000, 3, kc, True, y.ptr, kc)
    assert dev.history_len == h and dev.nsegments == kc
    for bad in (_AddressOnly((40, 3), F64), _AddressOnly((40, 4), F32), _AddressOnly((40,), F32)):
        with pytest.raises(dsp.ArgumentError):
            dev.stft(bad)
    x2 = _AddressOnly((600, 3), F32, _ptr=1 << 28)
    kc2, _ = stft_stream_step(h, 600, n, n - hop, True)
    for out in (_AddressOnly((n // 2 + 1, kc2 - 1, 3), F32),            # too few columns
                _AddressOnly((n // 2 + 1, kc2, 3), F64),                # wrong eltype
                _AddressOnly((n // 2, kc2, 3), F32),                    # wrong nout
                _AddressOnly((n // 2 + 1, kc2, 2), F32),                # wrong channel count
                _AddressOnly((n // 2 + 1, kc2, 3), F32, _ptr=(1 << 28) + 400),    # overlaps x
                _AddressOnly((n // 2 + 1, kc2, 3), F32, _ptr=hist_out + 8)):     # overlaps the history
        with pytest.raises(dsp.ArgumentError):
            dev.stft_(out, x2)
    with pytest.raises(dsp.ArgumentError):
        dev.stft_(np.zeros((n // 2 + 1, kc2, 3), F32, order="F"), x2)
    assert len(fake.calls) == 1 and dev.nsegments == kc
    out = _AddressOnly((n // 2 + 1, kc2 + 5, 3), F32)
    assert dev.stft_(out, x2) == kc2
    c2 = fake.calls[-1]
    assert c2[1] == hist_out and c2[2] == h and c2[11:13] == (out.ptr, kc2 + 5)          # histories swap
    assert dev.history.ptr == c2[3]
    # an empty chunk launches nothing
    ncalls = len(fake.calls)
    assert dev.stft(_AddressOnly((0, 3), F32)).shape == (n // 2 + 1, 0, 3) and len(fake.calls) == ncalls
    # finish(): the held-back segment (if any) unpaired, then chunks are refused until reset()
    held = dev.history_len >= n
    f = dev.finish()
    assert f.shape == (n // 2 + 1, 1 if held else 0, 3) and len(fake.calls) == ncalls + held
    if held:
        assert fake.calls[-1][5:9] == (None, 0, 3, 1)
    with pytest.raises(dsp.ArgumentError):
        dev.stft(x2)
    dev.reset()
    assert dev._key is None and dev.history is None and dev.nsegments == 0
    dev.stft(_AddressOnly((7,), F64))
    assert fake.calls[-1][1] is None


# =============================================================================== GPU

def _signal(rng, shape, dt):
    x = rng.standard_normal(shape)
    if dt.kind == "c":
        x = x + 1j * rng.standard_normal(shape)
    return np.asfortranarray(x.astype(dt))


def _oneshot(x, **kw):
    """stft of each channel on its own, one aligned vector each (the comparison target): (nout, k, nchan)."""
    cols = [dsp.stft(dsp.to_device(np.ascontiguousarray(x[:, c])), **kw).to_host() for c in range(x.shape[1])]
    return np.stack(cols, axis=2)


def _stream(x, sizes, device=True, **kw):
    """x streamed in chunks of the given lengths; returns the concatenated columns (nout, k, nchan)."""
    s = dsp.STFTStream(device=device, **kw)
    parts, a = [], 0
    for c in sizes:
        chunk = np.asfortranarray(x[a:a + c])
        a += c
        y = s.stft(dsp.to_device(chunk) if device else chunk)
        parts.append(y.to_host() if device else y)
    f = s.finish()
    parts.append(f.to_host() if device else f)
    return np.concatenate(parts, axis=1)


def _same(a, b):
    """Bit for bit (a +0 / -0 or NaN payload difference counts)."""
    return (a.shape == b.shape and a.dtype == b.dtype and
            np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes())


FUSED = [(F32, N) for N in (256, 512, 1024, 2048, 4096, 8192, 16384)] + [(F64, N) for N in (256, 1024, 8192)] + \
        [(C64, N) for N in (256, 1024, 4096, 16384)] + [(C128, N) for N in (512, 8192)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", FUSED, ids=[f"{d.name}-{N}" for d, N in FUSED])
def test_stream_is_bit_identical_every_fused_size(dt, N):
    rng = np.random.default_rng(N)
    hop = N // 2
    for psd, win, ones in ((True, dsp.hanning, None), (False, None, None), (True, None, False if dt.kind == "f" else None)):
        kw = dict(n=N, noverlap=N - hop, psdonly=psd, nfft=N, window=win, onesided=ones)
        x = _signal(rng, (5 * N + 37, 3), dt)
        want = _oneshot(x, **kw)
        for sizes in ([1 + 3 * hop // 2], [hop - 1], [hop], [hop + 1], [N - 1], [N], [N + hop], None):
            if sizes == [hop - 1] and N > 2048:
                continue                                          # thousands of launches: covered by the small sizes
            got = _stream(x, _chunk_sizes(rng, x.shape[0], sizes), **kw)
            assert _same(got, want), (dt, N, psd, win, ones, sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F64, C64])
def test_overlaps_padding_alignment_and_channels(dt):
    rng = np.random.default_rng(11)
    for n, nfft in ((1024, 1024), (1000, 1024), (400, 512), (4096, 4096)):
        for noverlap in (0, n // 2, 3 * n // 4, n - 1):
            kw = dict(n=n, noverlap=noverlap, psdonly=bool(noverlap % 2 == 0), nfft=nfft, window=dsp.hanning)
            hop = n - noverlap
            nch = 3 if noverlap != n // 2 else 70
            x = _signal(rng, (3 * n + 9 * hop + 5, nch), dt)
            want = _oneshot(x, **kw)
            # odd chunk lengths put the history at every alignment (thread-loaded units), random ones everywhere
            for sizes in ([hop + 1], [3, 5, 7], None):
                if hop == 1 and sizes != [3, 5, 7]:
                    continue
                got = _stream(x, _chunk_sizes(rng, x.shape[0], sizes), **kw)
                assert _same(got, want), (dt, n, nfft, noverlap, sizes)


@pytest.mark.gpu
def test_direct_load_path_float64_8192():
    # the Float64 8192-point stage does not fit with the transform's shared memory: units are read directly
    rng = np.random.default_rng(3)
    kw = dict(n=8192, noverlap=2048, psdonly=False, nfft=8192, window=dsp.hamming)
    x = _signal(rng, (6 * 8192 + 11, 1), F64)
    want = _oneshot(x, **kw)
    assert _same(_stream(x, _chunk_sizes(rng, x.shape[0], [5000, 8193, 1]), **kw), want)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,n,nfft", [(F32, 400, 400), (F32, 1000, 1000), (C64, 1000, 1000), (F64, 300, 320),
                                       (F32, 20000, 20000), (C128, 5000, 24000)])
def test_cufft_sizes(dt, n, nfft):
    rng = np.random.default_rng(n)
    for psd in (True, False):
        kw = dict(n=n, noverlap=n // 4, psdonly=psd, nfft=nfft, window=dsp.hanning)
        x = _signal(rng, (7 * n + 13, 3), dt)
        want = _oneshot(x, **kw)
        for sizes in ([n // 3], [n + 7], None):
            assert _same(_stream(x, _chunk_sizes(rng, x.shape[0], sizes), **kw), want), (dt, n, nfft, psd, sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", [(F32, 1024), (C64, 4096), (F32, 1000)])
def test_host_stream_equals_device_stream(dt, N):
    rng = np.random.default_rng(5)
    kw = dict(n=N, noverlap=3 * N // 4, psdonly=True, nfft=N, window=dsp.hanning)
    x = _signal(rng, (6 * N + 3, 3), dt)
    hs, ds = dsp.STFTStream(**kw), dsp.STFTStream(device=True, **kw)
    a = 0
    for c in _chunk_sizes(rng, x.shape[0], None):
        chunk = np.asfortranarray(x[a:a + c])
        a += c
        assert _same(hs.stft(chunk), ds.stft(dsp.to_device(chunk)).to_host())
        assert hs.history_len == ds.history_len and hs.nsegments == ds.nsegments
        if hs.history is not None:
            assert _same(np.asfortranarray(hs.history), np.asfortranarray(ds.history.to_host()[:ds.history_len]))
    assert _same(hs.finish(), ds.finish().to_host())


@pytest.mark.gpu
def test_c4_full_size_in_65536_sample_blocks():
    rng = np.random.default_rng(4)
    nchan, length = 64, 1 << 22
    x = rng.standard_normal((length, nchan)).astype(F32, order="F")
    kw = dict(n=1024, noverlap=768, psdonly=True, nfft=1024, window=dsp.hanning)
    dx = dsp.to_device(x)
    want = dsp.stft(dx, **kw).to_host()                          # one-shot matrix call (aligned: the warp plan)
    s = dsp.STFTStream(device=True, **kw)
    parts = []
    for a in range(0, length, 65536):
        parts.append(s.stft(dsp.to_device(np.asfortranarray(x[a:a + 65536]))).to_host())
    parts.append(s.finish().to_host())
    assert _same(np.concatenate(parts, axis=1), want)


@pytest.mark.gpu
def test_spectrogram_time_axes():
    rng = np.random.default_rng(8)
    x = _signal(rng, (20000,), F32)
    ref = dsp.spectrogram(x, 512, 384, fs=8000.0, window=dsp.hanning)
    s = dsp.STFTStream(512, 384, psdonly=True, fs=8000.0, window=dsp.hanning, device=True)
    ts, ps = [], []
    for a in range(0, x.size, 3001):
        sp = s.spectrogram(dsp.to_device(x[a:a + 3001]))
        ts.append(sp.time)
        ps.append(sp.power.to_host())
        assert np.array_equal(sp.freq, ref.freq)
    f = s.finish()
    if f.shape[1]:
        ts.append(s._times(s.nsegments - 1, 1))
        ps.append(f.to_host())
    assert np.array_equal(np.concatenate(ts), ref.time)
    assert _same(np.concatenate(ps, axis=1), ref.power)


@pytest.mark.gpu
def test_launch_counts():
    rng = np.random.default_rng(9)
    for dt, n in ((F32, 1024), (F32, 512), (C64, 2048)):
        s = dsp.STFTStream(n, psdonly=True, window=dsp.hanning, device=True)
        for c in (1, 700, n - 1, 3 * n + 5, 65536):
            x = dsp.to_device(_signal(rng, (c, 5), dt))
            before = dsp.launch_count()
            s.stft(x)
            assert dsp.launch_count() - before <= 2
        before = dsp.launch_count()
        s.stft(dsp.to_device(np.zeros((0, 5), dt, order="F")))
        assert dsp.launch_count() == before


@pytest.mark.gpu
def test_c_abi_refuses_overlaps_before_any_launch():
    n, hop, nch = 256, 128, 2
    plan = _lib.SpecPlan(F32, n, n - hop, n, True, None)
    ldh, nx, nseg, nout = n + hop - 1, 1000, 6, n // 2 + 1
    hist_in, hist_out = DeviceArray((ldh, nch), F32), DeviceArray((ldh, nch), F32)
    x, out = DeviceArray((nx, nch), F32), DeviceArray((nout, nseg, nch), F32)
    good = (hist_in.ptr, 0, hist_out.ptr, ldh, x.ptr, nx, nch, nseg, 1.0, True, out.ptr, nseg)
    before = dsp.launch_count()
    bad = [
        {2: hist_in.ptr},                                       # hist_out == hist_in
        {2: x.ptr},                                             # hist_out overlaps x
        {2: out.ptr + 64},                                      # hist_out overlaps out
        {10: x.ptr + 4},                                        # out overlaps x
        {10: hist_in.ptr},                                      # out overlaps hist_in
        {11: nseg - 1},                                         # ldo < nseg
        {7: nseg + 2},                                          # segments past the virtual column
        {3: 100},                                               # the new history exceeds ldh
        {1: 10, 0: None},                                       # nhist > 0 without hist_in
    ]
    for b in bad:
        args = list(good)
        for i, v in b.items():
            args[i] = v
        with pytest.raises(_lib.DSPB200Error):
            plan.stft_stream_dev(*args)
    assert dsp.launch_count() == before
    plan.stft_stream_dev(*good)
    dsp.sync()
    assert 1 <= dsp.launch_count() - before <= 2
