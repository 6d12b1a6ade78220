"""Host-pointer entry points against their device-pointer twins.

Every host form (`dspb200_*_exec`) stages its buffers around the device form (`dspb200_*_exec_dev`), so on the same data
the two must agree bit for bit.  Also checked here: the stateful host forms filtering in place, the empty cases that
return before any launch, and that a host form which fails after staging (an unsupported stateful overlap-save plan)
leaves the library usable for the next call."""
import numpy as np
import pytest

from dspb200 import _lib
from dspb200.device import DeviceArray, to_device

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64, np.complex64, np.complex128]
UINT = {4: np.uint32, 8: np.uint64, 16: np.uint64}


def _signal(rng, shape, dt):
    x = rng.standard_normal(shape)
    if np.dtype(dt).kind == "c":
        x = x + 1j * rng.standard_normal(shape)
    return np.asfortranarray(x.astype(dt))


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(UINT[a.dtype.itemsize])


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(_bits(a), _bits(b))


def _dev_empty(shape, dt):
    return DeviceArray(shape, dt)


@pytest.mark.parametrize("dt", DTYPES)
def test_stft_host_matches_device(dt):
    rng = np.random.default_rng(1)
    onesided = np.dtype(dt).kind != "c"
    for nfft in (256, 1000):                              # fused and cuFFT sizes
        plan = _lib.SpecPlan(dt, 200, 100, nfft, onesided, np.hanning(200))
        n, nchan = 2000, 3
        s = _signal(rng, (n, nchan), dt)
        k = plan.nsegments(n)
        for psd in (True, False):
            odt = np.dtype(dt).type(0).real.dtype if psd else np.result_type(dt, np.complex64)
            host = np.zeros((plan.nout, k * nchan), dtype=odt, order="F")
            plan.stft(s, n, nchan, 2.0, psd, host)
            d_out = _dev_empty((plan.nout, k * nchan), odt)
            plan.stft_dev(to_device(s).ptr, n, nchan, 2.0, psd, d_out.ptr)
            assert _same(host, d_out.to_host())


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_multitaper_host_matches_device(dt):
    rng = np.random.default_rng(2)
    n = 512
    tapers = np.stack([np.hanning(n), np.hamming(n), np.blackman(n)]) / 10.0
    for nfft in (512, 600):
        plan = _lib.MtPlan(dt, n, 0, nfft, True, tapers)
        s = _signal(rng, (n,), dt)
        host = np.zeros(plan.nout, dtype=dt)
        plan.mt_pgram(s, host)
        d_out = _dev_empty((plan.nout,), dt)
        plan.mt_pgram_dev(to_device(s).ptr, n, d_out.ptr)
        assert _same(host, d_out.to_host())
        plan = _lib.MtPlan(dt, 128, 64, nfft, True, np.stack([np.hanning(128), np.hamming(128)]))
        s = _signal(rng, (1000,), dt)
        k = plan.nsegments(s.size)
        host = np.zeros((plan.nout, k), dtype=dt, order="F")
        plan.mt_spectrogram(s, host)
        d_out = _dev_empty((plan.nout, k), dt)
        plan.mt_spectrogram_dev(to_device(s).ptr, s.size, d_out.ptr)
        assert _same(host, d_out.to_host())
        short = np.zeros(10, dtype=dt)                        # no segment: nothing written
        out = np.full(4, 7, dtype=dt)
        plan.mt_spectrogram(short, out)
        assert np.all(out == 7)


@pytest.mark.parametrize("dt", DTYPES)
def test_fir_and_overlap_save_host_match_device(dt):
    rng = np.random.default_rng(3)
    nx, ncols = 3000, 2
    x = _signal(rng, (nx, ncols), dt)
    b = _signal(rng, (37,), dt).ravel()
    fp = _lib.FirPlan(b)
    host = np.zeros_like(x)
    fp.exec(x, host)
    d_out = _dev_empty((nx, ncols), dt)
    fp.exec_dev(to_device(x).ptr, nx, ncols, d_out.ptr)
    assert _same(host, d_out.to_host())
    for nfft in (0, 4096 + 8):                              # fused and cuFFT
        op = _lib.OsPlan(b, nfft)
        nout = nx + b.size - 1
        host = np.zeros((nout, ncols), dtype=dt, order="F")
        op.exec(x, host, nx, ncols, nout)
        d_out = _dev_empty((nout, ncols), dt)
        op.exec_dev(to_device(x).ptr, nx, ncols, d_out.ptr, nout)
        assert _same(host, d_out.to_host())
        zeros = np.full((5, 2), 3, dtype=dt, order="F")     # nu == 0: zeros
        op.exec(np.zeros((0, 2), dtype=dt), zeros, 0, 2, 5)
        assert np.all(zeros == 0)
        untouched = np.full(5, 3, dtype=dt)                 # ncols == 0: nothing written
        op.exec(x, untouched, nx, 0, 5)
        fp.exec(np.zeros((nx, 0), dtype=dt), untouched)
        assert np.all(untouched == 3)


@pytest.mark.parametrize("dt", DTYPES)
def test_resample_host_matches_device(dt):
    rng = np.random.default_rng(4)
    h = rng.standard_normal(48).astype(np.float32)
    plan = _lib.ResamplePlan(dt, h, 3, 2)
    nx, ncols = 1000, 2
    x = _signal(rng, (nx, ncols), dt)
    nout = 1400
    host = np.zeros((nout, ncols), dtype=plan.out_dtype, order="F")
    plan.exec(x, nx, ncols, 0, 0, host, nout)
    d_out = _dev_empty((nout, ncols), plan.out_dtype)
    plan.exec_dev(to_device(x).ptr, nx, ncols, 0, 0, d_out.ptr, nout)
    assert _same(host, d_out.to_host())
    untouched = np.full(4, 3, dtype=plan.out_dtype)          # nout == 0 / ncols == 0: nothing written
    plan.exec(x, nx, ncols, 0, 0, untouched, 0)
    plan.exec(x, nx, 0, 0, 0, untouched, nout)
    assert np.all(untouched == 3)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("kind", ["fir", "os"])
def test_stateful_host_forms_in_place_and_empty(dt, kind):
    rng = np.random.default_rng(5)
    b = _signal(rng, (29,), dt).ravel()
    plan = _lib.FirPlan(b) if kind == "fir" else _lib.OsPlan(b)
    ns, nx, ncols = b.size - 1, 2500, 3
    x = _signal(rng, (nx, ncols), dt)
    si = _signal(rng, (ns, ncols), dt)
    out = np.zeros_like(x)
    so = np.zeros_like(si)
    plan.exec_state(x, nx, ncols, si, so, out)
    d_out, d_so = _dev_empty((nx, ncols), dt), _dev_empty((ns, ncols), dt)
    plan.exec_state_dev(to_device(x).ptr, nx, ncols, to_device(si).ptr, d_so.ptr, d_out.ptr)
    assert _same(out, d_out.to_host()) and _same(so, d_so.to_host())
    xi, sii = x.copy(order="F"), si.copy(order="F")        # out is x, si_out is si_in
    plan.exec_state(xi, nx, ncols, sii, sii, xi)
    assert _same(xi, out) and _same(sii, so)
    z = np.full_like(si, 5)                                 # nx == 0, si_in NULL: zero state
    plan.exec_state(np.zeros((0, ncols), dtype=dt), 0, ncols, None, z, np.zeros((0, ncols), dtype=dt))
    assert np.all(z == 0)
    p = np.zeros_like(si)                                   # nx == 0, si_in set: passed through
    plan.exec_state(np.zeros((0, ncols), dtype=dt), 0, ncols, si, p, np.zeros((0, ncols), dtype=dt))
    assert _same(p, si)
    d_p = _dev_empty((ns, ncols), dt)
    plan.exec_state_dev(None, 0, ncols, to_device(si).ptr, d_p.ptr, None)
    assert _same(d_p.to_host(), si)


def test_unsupported_stateful_plan_leaves_the_next_call_correct():
    rng = np.random.default_rng(6)
    v = rng.standard_normal(33).astype(np.float32)
    bad = _lib.OsPlan(v, 512)
    assert bad.fused
    x = _signal(rng, (4000, 2), np.float32)
    si = _signal(rng, (v.size - 1, 2), np.float32)
    with pytest.raises(_lib.DSPB200Error):
        bad.exec_state(x, 4000, 2, si, np.zeros_like(si), np.zeros_like(x))
    good, ref = _lib.OsPlan(v), _lib.FirPlan(v)
    out, so = np.zeros_like(x), np.zeros_like(si)
    good.exec_state(x, 4000, 2, si, so, out)
    out_fir, so_fir = np.zeros_like(x), np.zeros_like(si)
    ref.exec_state(x, 4000, 2, si, so_fir, out_fir)
    assert np.allclose(out, out_fir, rtol=1e-4, atol=1e-4) and np.allclose(so, so_fir, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("dt", DTYPES)
def test_welch_batch_shorter_than_one_segment(dt):
    onesided = np.dtype(dt).kind != "c"
    plan = _lib.SpecPlan(dt, 256, 128, 256, onesided, np.hanning(256))
    rdt = np.dtype(dt).type(0).real.dtype
    s = np.ones((100, 2), dtype=dt, order="F")
    host = np.full((plan.nout, 2), 9, dtype=rdt, order="F")
    plan.welch_batch(s, 100, 2, 1.0, host)
    assert np.all(host == 0)
    d_out = to_device(np.full((plan.nout, 2), 9, dtype=rdt, order="F"))
    plan.welch_batch_dev(to_device(s).ptr, 100, 2, 1.0, d_out.ptr)
    assert np.all(d_out.to_host() == 0)
