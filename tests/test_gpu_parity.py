"""GPU parity: the CUDA path (through the C ABI, via the host mirror `dspb200`) against the CPU oracle, the
reference's golden vectors and its known-answer tests.  Mirrors the reference's own tests (file:line cited).

Tolerances (BASELINE.json north_star): norm-relative 1e-6 for Float32/ComplexF32, 1e-12 for Float64/ComplexF64,
measured against the double-precision oracle (SURVEY.md section 7, hard part 2)."""
from fractions import Fraction

import numpy as np
import pytest

from conftest import approx, relerr

pytestmark = pytest.mark.gpu

dsp = pytest.importorskip("dspb200")
from oracle import dspbase as od          # noqa: E402
from oracle import filters as of          # noqa: E402
from oracle import periodograms as op     # noqa: E402
from oracle import windows as ow          # noqa: E402

TOL32 = 1e-6
TOL64 = 1e-12
# (every bound that was once widened -- 2 * TOL, 2e-6, 5e-6, 1e-11 -- is back at the north_star value and holds on an H100)
RNG = np.random.default_rng(1776)


def tol(dt):
    return TOL32 if np.dtype(dt) in (np.dtype(np.float32), np.dtype(np.complex64)) else TOL64


def randn(n, dt):
    dt = np.dtype(dt)
    if dt.kind == "c":
        return (RNG.standard_normal(n) + 1j * RNG.standard_normal(n)).astype(dt)
    return RNG.standard_normal(n).astype(dt)


# =============================================================================== filt(b, a, x)

def test_filt_exact_small():
    # test/dsp.jl:10-21, 34
    b = np.array([1., 2., 3., 4.])
    x = np.array([1., 1., 0., 1., 1., 0., 0., 0.])
    assert np.array_equal(dsp.filt(b, 1., x), [1., 3., 5., 8., 7., 5., 7., 4.])
    assert np.array_equal(dsp.filt(b, 1., np.arange(1.0, 11.0)), [1., 4., 10., 20., 30., 40., 50., 60., 70., 80.])
    assert np.array_equal(dsp.filt(np.arange(1.0, 5.0), 1., np.arange(1.0, 11.0)), [1., 4., 10., 20., 30., 40., 50., 60., 70., 80.])
    x2 = np.stack([x, np.arange(1.0, 9.0)], axis=1)
    y2 = dsp.filt(b, 1., x2)
    assert np.array_equal(y2[:, 0], dsp.filt(b, 1., x)) and np.array_equal(y2[:, 1], dsp.filt(b, 1., np.arange(1.0, 9.0)))
    with pytest.raises(dsp.ArgumentError):
        dsp.filt_(np.zeros(2), [1.], [1.], [1.])
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(np.zeros(0), 1., x)
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(b, 0., x)
    assert np.array_equal(dsp.filt([2.0], 4.0, x), x * 0.5)        # max(na, nb) == 1: plain scaling, :40


@pytest.mark.parametrize("dt", [np.float32, np.float64, np.complex64, np.complex128])
@pytest.mark.parametrize("nb", [2, 19, 66, 67, 257, 1500])
def test_filt_fir_matches_reference_order(dt, nb):
    # config 1 shape (257 taps) and the SMALL_FILT_CUTOFF boundary; the kernel reproduces the reference's
    # oldest-tap-first fma chain, so real Float32/Float64 results are bit-identical to the restated loop.
    b = randn(nb, dt)
    x = randn(5000, dt)
    y = dsp.filt(b, np.ones(1, dtype=dt), x)
    ref = od.filt(b, np.ones(1, dtype=dt), x)
    assert y.dtype == np.dtype(dt) and y.shape == x.shape
    if np.dtype(dt) == np.float32:
        assert np.array_equal(y, ref)
    truth = od.filt(b, np.ones(1, dtype=dt), x, f64=True)
    assert relerr(y, truth) <= max(relerr(ref, truth) * 1.01, tol(dt))


def test_filt_columns_and_normalisation():
    # test/filt.jl:71-93: trailing dims are independent channels; a[1] != 1 normalises b (:43-47)
    b = randn(7, np.float64)
    x = randn(300 * 6, np.float64).reshape(300, 2, 3)
    y = dsp.filt(b, 2.0, x)
    for i in range(2):
        for j in range(3):
            assert np.array_equal(y[:, i, j], dsp.filt(b, 2.0, x[:, i, j]))
    assert relerr(y[:, 1, 2], od.filt(b / 2.0, 1.0, x[:, 1, 2])) < 1e-15


def test_config1_full_size():
    # BASELINE config 1: 257-tap FIR on 2^20 Float32, full size against the oracle restatement (bit-exact)
    n = np.arange(257) - 128
    b = (0.5 * np.sinc(0.5 * n) * np.hamming(257)).astype(np.float32)
    x = np.random.default_rng(1001).standard_normal(1 << 20).astype(np.float32)
    y = dsp.filt(b, np.float32(1), x)
    assert np.array_equal(y, od.filt(b, np.ones(1, np.float32), x))


# =============================================================================== fftfilt / filt(b, x) / tdfilt

@pytest.mark.parametrize("xlen", [2 ** 7 - 1, 2 ** 10 - 1, 2 ** 13 - 1, 2 ** 16 - 1, 2 ** 18 - 1])
@pytest.mark.parametrize("blen", [2 ** 1 - 1, 2 ** 4 - 1, 2 ** 7 - 1])
def test_fftfilt_filt_tdfilt_agree(xlen, blen):
    # test/filt.jl:312-331
    b = randn(blen, np.float64)
    for x in (randn(xlen, np.float64), randn(xlen * 2, np.float64).reshape(xlen, 2)):
        ref = dsp.filt(b, [1.0], x)
        assert approx(dsp.fftfilt(b, x), ref)
        assert approx(dsp.filt(b, x), ref)
        assert approx(dsp.tdfilt(b, x), ref)
        out = np.empty_like(x)
        assert approx(dsp.fftfilt_(out, b, x), ref)
        assert approx(dsp.tdfilt_(out, b, x), ref)
        assert relerr(dsp.fftfilt(b, x), od.filt(b, [1.0], x, f64=True)) < TOL64
    with pytest.raises(dsp.ArgumentError):
        dsp.fftfilt_(np.empty(3), b, randn(xlen, np.float64))


@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("nb,nx,nfft", [(257, 1 << 20, None), (257, 1 << 20, 2048), (67, 100000, 512),
                                         (1000, 77777, None), (4097, 1 << 18, None), (9000, 1 << 17, None),
                                         (300, 5000, 1000), (129, 4000, 16384)])
def test_fftfilt_sizes(dt, nb, nx, nfft):
    # fused power-of-two blocks, explicit reference-style nfft, the cuFFT path (non power of two / long taps)
    if np.dtype(dt) == np.float64 and nfft == 16384:
        nfft = 8192
    b = randn(nb, dt)
    x = randn(nx, dt)
    y = dsp.fftfilt(b, x, nfft)
    assert y.dtype == np.dtype(dt) and y.shape == x.shape
    assert relerr(y, od.filt(b, np.ones(1, dtype=dt), x, f64=True)) < tol(dt)


# =============================================================================== conv

def test_conv_exact_integers_and_empty():
    # test/dsp.jl:41-59, 80-81
    a = np.array([1, 2, 1, 2])
    b = np.array([1, 2, 3])
    exp = [1, 4, 8, 10, 7, 6]
    assert np.array_equal(dsp.conv(a, b), exp)
    assert np.array_equal(dsp.conv(a.astype(np.int32), b), exp)
    assert np.array_equal(dsp.conv(a.astype(float), b.astype(float)), exp)
    assert np.array_equal(dsp.conv(a * 1j, b.astype(complex)).imag, exp)
    for alg in ("direct", "fft", "fft_simple", "fft_overlapsave"):
        assert np.array_equal(dsp.conv(randn(5, np.float64), np.zeros(0), algorithm=alg), np.zeros(4))
        assert dsp.conv(np.zeros(0), np.zeros(0), algorithm=alg).size == 0


@pytest.mark.parametrize("dt", [np.float64, np.complex128, np.float32, np.complex64])
def test_conv_algorithms_agree(dt):
    # test/dsp.jl:72-77, 98-121
    for M in (10, 200):
        for N in (10, 200):
            u, v = randn(M, dt), randn(N, dt)
            ref = dsp.conv(u, v, algorithm="direct")
            assert relerr(ref, od.conv_exact(u, v)) < tol(dt)
            for alg in ("fft_simple", "fft_overlapsave", "fft", "fast", "auto"):
                y = dsp.conv(u, v, algorithm=alg)
                assert y.dtype == np.dtype(dt)
                assert approx(y, ref), (M, N, alg)
                assert relerr(y, od.conv_exact(u, v)) < tol(dt), (M, N, alg)
    with pytest.raises(dsp.ArgumentError):
        dsp.conv(np.ones(300), np.ones(300), algorithm="bogus")
    # over-sized out is zero-filled (test/dsp.jl:109-112)
    u, v = randn(200, dt), randn(10, dt)
    out = np.full(300, 7, dtype=dt)
    dsp.conv_(out, u, v, algorithm="fft_overlapsave")
    assert approx(out[:209], dsp.conv(u, v)) and not out[209:].any()


@pytest.mark.parametrize("dt", [np.float32, np.float64, np.complex128, np.complex64])
@pytest.mark.parametrize("nu,nv,nfft", [(128, 12, None), (128, 128, None), (128, 12, 256), (128, 13, 32),
                                         (128, 12, 32), (25, 4, 16), (128, 12, 140), (1000, 33, 64)])
def test_os_kernel_vs_single_fft(dt, nu, nv, nfft):
    # test/dsp.jl:271-314 (N = 1): regular, adversarial (nsmall, nfft) and the "three padded blocks" case
    u, v = randn(nu, dt), randn(nv, dt)
    os_out = dsp.conv(u, v, algorithm="fft_overlapsave", nfft=nfft)
    single = dsp.conv(u, v, algorithm="fft_simple")
    assert os_out.dtype == np.dtype(dt)
    assert approx(os_out, single)
    assert relerr(os_out, od.conv_exact(u, v)) < tol(dt)
    assert relerr(single, od.conv_exact(u, v)) < tol(dt)


@pytest.mark.parametrize("dt", [np.complex64, np.float32, np.complex128, np.float64])
def test_conv_config2_scaled(dt):
    # BASELINE config 2 shape at 2^20: 4097-tap FIR, overlap-save (library-chosen block and the reference's 65536)
    nv, nu = 4097, 1 << 20
    n = np.arange(nv) - nv // 2
    v = (0.2 * np.sinc(0.2 * n) * np.hamming(nv))
    v = (v * np.exp(1j * np.pi * 0.3 * n)).astype(dt) if np.dtype(dt).kind == "c" else v.astype(dt)
    u = randn(nu, dt)
    truth = od.conv_exact(u, v)
    for nfft in (None, 65536, 8192):
        y = dsp.conv(u, v, algorithm="fft_overlapsave", nfft=nfft)
        assert y.dtype == np.dtype(dt) and y.size == nu + nv - 1
        assert relerr(y, truth) < tol(dt), nfft
    ref32 = od.conv_kern_os(u, v, 65536)                   # the reference's own arithmetic (same dtype, nfft 65536)
    assert relerr(y, truth) <= max(2 * relerr(ref32, truth), tol(dt))


def test_conv_config2_full_size_probes():
    # BASELINE config 2 at full size (2^26 ComplexF32, 4097 taps): direct double-precision evaluation of the
    # convolution sum at 2000 probe outputs (incl. both edges and block boundaries), plus linearity.
    nv, nu = 4097, 1 << 26
    rng = np.random.default_rng(1002)
    u = np.empty(nu, dtype=np.complex64)
    for i in range(0, nu, 1 << 22):
        u[i:i + (1 << 22)] = ((rng.standard_normal(1 << 22) + 1j * rng.standard_normal(1 << 22)) / np.sqrt(2)).astype(np.complex64)
    n = np.arange(nv) - nv // 2
    v = (0.2 * np.sinc(0.2 * n) * np.hamming(nv) * np.exp(1j * np.pi * 0.3 * n)).astype(np.complex64)
    y = dsp.conv(u, v, algorithm="fft_overlapsave")
    assert y.size == nu + nv - 1
    L = 16384 - nv + 1
    probes = np.concatenate([np.arange(0, 40), np.arange(nu + nv - 41, nu + nv - 1), np.arange(L - 20, L + 20),
                             np.arange(1000 * L - 20, 1000 * L + 20), rng.integers(0, nu + nv - 1, 1800)])
    v64 = v.astype(np.complex128)
    ref = np.empty(probes.size, dtype=np.complex128)
    for i, m in enumerate(probes):
        lo, hi = max(0, m - nv + 1), min(nu - 1, m)
        ref[i] = np.dot(u[lo:hi + 1].astype(np.complex128), v64[m - lo - np.arange(hi - lo + 1)])
    scale = np.sqrt(np.mean(np.abs(ref) ** 2))
    assert np.sqrt(np.mean(np.abs(y[probes] - ref) ** 2)) / scale < TOL32
    # linearity on a slice: conv(2u) == 2 conv(u) exactly in floating point (power-of-two scale)
    y2 = dsp.conv(2 * u[: 1 << 22], v, algorithm="fft_overlapsave")
    assert np.array_equal(y2[: 1 << 21], 2 * y[: 1 << 21])


# =============================================================================== periodogram / Welch

DATA = np.arange(8)
DATA0 = np.array([98.0, 13.656854249492380, 4.0, 2.343145750507620, 2.0, 2.343145750507620, 4.0, 13.656854249492380])


def test_periodogram_welch_spectrogram_0to7():
    # test/periodograms.jl:92-106
    assert approx(dsp.periodogram(DATA, onesided=False).power, DATA0)
    with pytest.warns(DeprecationWarning):
        assert approx(dsp.welch_pgram(DATA, 8, 0, onesided=False).power, DATA0)
    assert approx(dsp.welch_pgram(DATA, 8, 0, onesided=False, window=None).power, DATA0)
    assert approx(dsp.spectrogram(DATA, 8, 0, onesided=False).power[:, 0], DATA0)
    z = DATA + 1j * DATA
    assert approx(dsp.periodogram(z, onesided=False).power, DATA0 * 2)
    assert approx(dsp.welch_pgram(z, 8, 0, onesided=False, window=None).power, DATA0 * 2)
    assert approx(dsp.spectrogram(z, 8, 0, onesided=False).power[:, 0], DATA0 * 2)
    with pytest.raises(dsp.ArgumentError):
        dsp.periodogram(z, onesided=True)
    with pytest.raises(dsp.DomainError):
        dsp.periodogram(DATA, nfft=4)


@pytest.mark.parametrize("n,nov,expected", [(2, 0, [34.5, 0.5]), (3, 0, [25.5, 1.0, 1.0]),
                                            (3, 1, [35.0, 1.0, 1.0]), (4, 1, [45, 2, 1, 2])])
def test_welch_rect_kats(n, nov, expected):
    # test/periodograms.jl:108-131 (MATLAB pwelch)
    assert approx(dsp.welch_pgram(DATA, n, nov, onesided=False, window=None).power, np.array(expected, float))
    assert approx(dsp.spectrogram(DATA, n, nov, onesided=False).power.mean(axis=1), np.array(expected, float))


def test_windowed_and_padded_periodogram_kats():
    # test/periodograms.jl:139-222
    cases = ((dsp.hamming, [65.461623986801527, 20.556791795515764, 0.369313143650544, 0.022167446610882,
                            0.025502985564107, 0.022167446610882, 0.369313143650544, 20.556791795515764]),
             (dsp.bartlett, [62.999999999999993, 21.981076052592442, 0.285714285714286, 0.161781090264695,
                             0.142857142857143, 0.161781090264695, 0.285714285714286, 21.981076052592442]))
    for win, exp in cases:
        exp = np.array(exp)
        for w in (win, win(8)):
            assert approx(dsp.periodogram(DATA, window=w, onesided=False).power, exp, rtol=1e-8)
            assert approx(dsp.welch_pgram(DATA, 8, 0, window=w, onesided=False).power, exp, rtol=1e-8)
            assert approx(dsp.spectrogram(DATA, 8, 0, window=w, onesided=False).power[:, 0], exp, rtol=1e-8)
    exp = np.array([98, 174.463067389405, 121.968086934209, 65.4971744936088, 27.3137084989848, 12.1737815028909,
                    10.3755170959439, 10.4034038628775, 8, 5.25810953219633, 4.47015397150535, 4.89522578856669,
                    4.68629150101524, 3.69370284475603, 3.1862419983415, 3.61553458569862, 2])
    assert approx(dsp.periodogram(DATA, nfft=32).power, exp)
    assert approx(dsp.welch_pgram(DATA, 8, 0, nfft=32, window=None).power, exp)
    assert approx(dsp.spectrogram(DATA, 8, 0, nfft=32).power[:, 0], exp)
    exph = np.array([65.4616239868015, 122.101693164395, 98.8444689598445, 69.020252632913, 41.1135835910315,
                     20.5496474310966, 8.43291449161938, 2.78001620362588, 0.738626287301088, 0.174995741770789,
                     0.0501563022944516, 0.0327357460012861, 0.0443348932217643, 0.0553999745503552,
                     0.0561319901616643, 0.0526025934871384, 0.0255029855641069])
    assert approx(dsp.periodogram(DATA, window=dsp.hamming, nfft=32).power, exph)
    assert approx(dsp.welch_pgram(DATA, 8, 0, window=dsp.hamming, nfft=32).power, exph)
    assert approx(dsp.spectrogram(DATA, 8, 0, window=dsp.hamming, nfft=32).power[:, 0], exph)


def test_welch_config_and_inplace():
    # test/periodograms.jl:224-237
    expected = dsp.welch_pgram(DATA, 8, 0, window=dsp.hamming, nfft=32).power
    config = dsp.WelchConfig(DATA, n=8, noverlap=0, window=dsp.hamming, nfft=32)
    assert np.array_equal(dsp.welch_pgram(DATA, config).power, expected)
    out = np.empty_like(expected)
    assert np.array_equal(dsp.welch_pgram_(out, DATA, config).power, expected)
    assert np.array_equal(dsp.welch_pgram_(out, DATA, 8, 0, window=dsp.hamming, nfft=32).power, expected)
    with pytest.raises(dsp.ArgumentError):
        dsp.welch_pgram_(out.astype(np.float32), DATA, config)
    with pytest.raises(dsp.ArgumentError):
        dsp.welch_pgram_(out.astype(np.float32), DATA.astype(np.float32), config)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.welch_pgram_(np.empty(0), DATA, config)
    assert np.array_equal(dsp.welch_pgram_(out, DATA.astype(np.float64), config).power, expected)
    config2 = dsp.WelchConfig(8, np.float64, n=8, noverlap=0, window=dsp.hamming, nfft=32)
    assert np.array_equal(dsp.welch_pgram(DATA.astype(float), config2).power, expected)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.welch_pgram(DATA, 8, 0, window=np.ones(7))
    with pytest.raises(dsp.DomainError):
        dsp.welch_pgram(DATA, 4, 4, window=None)


def test_spectrogram_matlab_golden(goldens):
    # test/periodograms.jl:25-36
    spec = dsp.spectrogram(goldens["spectrogram_x"], 256, 128, fs=10)
    assert approx(dsp.power(spec), goldens["spectrogram_p"])
    assert approx(dsp.freq(spec), goldens["spectrogram_f"])
    assert approx(dsp.time(spec), goldens["spectrogram_t"])
    assert relerr(spec.power, goldens["spectrogram_p"]) < TOL64


def test_stft_matlab_golden(goldens):
    # test/periodograms.jl:332-344 (fused 512-point path) and the same through cuFFT (nfft = 500)
    S = dsp.stft(goldens["stft_x"], 400, 400 - 160, nfft=512, fs=16000, window=dsp.hanning)
    Sml = goldens["stft_S_real"] + 1j * goldens["stft_S_imag"]
    assert S.shape == (257, 29) and S.dtype == np.complex128
    assert approx(S, Sml)
    assert relerr(S, Sml) < TOL64
    S500 = dsp.stft(goldens["stft_x"], 400, 240, nfft=500, window=dsp.hanning)
    assert relerr(S500, op.stft(goldens["stft_x"], 400, 240, nfft=500, window=ow.hanning)) < TOL64


@pytest.mark.parametrize("dt", [np.float32, np.float64, np.complex64, np.complex128])
@pytest.mark.parametrize("n,nov,nfft,onesided,win", [
    (256, 128, 256, None, "hanning"), (4096, 2048, 4096, None, "hanning"), (1024, 768, 1024, None, None),
    (1000, 300, 1024, False, "hamming"), (400, 240, 500, None, "hanning"), (4096, 0, 8192, None, None),
    (300, 299, 16384, None, "hanning"), (63, 17, 70, None, "hamming"), (5000, 2500, 32768, False, None),
    (2048, 1024, 2048, False, "hanning")])
def test_welch_stft_spectrogram_vs_oracle(dt, n, nov, nfft, onesided, win):
    # fused (power-of-two) and cuFFT (other sizes) paths; one/two-sided; odd and even segment counts
    cplx = np.dtype(dt).kind == "c"
    if cplx and onesided is None:
        onesided = False
    if np.dtype(dt) in (np.dtype(np.float64), np.dtype(np.complex128)) and nfft == 16384:
        nfft = 8192
    hop = n - nov
    for extra in (0, 1):
        length = n + hop * (37 + extra) + 5
        x = randn(length, dt)
        x = x + (np.cos(0.3 * np.arange(length)) * 3).astype(np.float32)
        x = x.astype(dt)
        w_d = {None: None, "hanning": dsp.hanning, "hamming": dsp.hamming}[win]
        w_o = {None: None, "hanning": ow.hanning, "hamming": ow.hamming}[win]
        p = dsp.welch_pgram(x, n, nov, onesided=onesided, nfft=nfft, fs=2.5, window=w_d)
        pr, fr = op.welch_pgram(x, n, nov, onesided=onesided, nfft=nfft, fs=2.5, window=w_o, f64=True)
        assert p.power.dtype == dsp.fftabs2type(dt) and p.power.shape == pr.shape
        assert relerr(p.power, pr) < tol(dt)
        assert np.allclose(p.freq, fr)
        sp = dsp.spectrogram(x, n, nov, onesided=onesided, nfft=nfft, fs=2.5, window=w_d)
        spr, _, tr = op.spectrogram(x, n, nov, onesided=onesided, nfft=nfft, fs=2.5, window=w_o, f64=True)
        assert sp.power.shape == spr.shape and sp.power.dtype == dsp.fftabs2type(dt)
        assert relerr(sp.power, spr) < tol(dt)
        assert np.allclose(sp.time, tr)
        S = dsp.stft(x, n, nov, onesided=onesided, nfft=nfft, window=w_d)
        Sr = op.stft(x, n, nov, onesided=onesided, nfft=nfft, window=w_o, f64=True)
        assert S.dtype == dsp.fftouttype(dt) and S.shape == Sr.shape
        assert relerr(S, Sr) < tol(dt)


def test_welch_config3_scaled_and_reference_budget():
    # BASELINE config 3 shape at 2^22: nfft = 4096, 50 % overlap, hanning, Float32.  The GPU error against the
    # double-precision truth must be within 1e-6 AND no worse than the reference's own sequential-Float32 path.
    rng = np.random.default_rng(1003)
    n = 1 << 22
    t = np.arange(n)
    x = (rng.standard_normal(n) + np.cos(2 * np.pi * 0.1 * t) + 0.1 * np.cos(2 * np.pi * 0.2345 * t)).astype(np.float32)
    p = dsp.welch_pgram(x, 4096, 2048, window=dsp.hanning)
    truth, _ = op.welch_pgram(x, 4096, 2048, window=ow.hanning, f64=True)
    ref32, _ = op.welch_pgram(x, 4096, 2048, window=ow.hanning, sequential=True)
    e_gpu, e_ref = relerr(p.power, truth), relerr(ref32, truth)
    assert p.power.dtype == np.float32
    assert e_gpu < TOL32 and e_gpu <= 1.5 * e_ref + 1e-7


def test_welch_config3_full_size_parseval():
    # BASELINE config 3 at full size (2^26 Float32): Parseval -- the one-sided PSD integrates to the mean
    # windowed segment power -- and the tone bins against a double-precision evaluation of those bins alone.
    rng = np.random.default_rng(1003)
    n, nseg, hop = 1 << 26, 4096, 2048
    x = np.empty(n, dtype=np.float32)
    for i in range(0, n, 1 << 22):
        t = np.arange(i, i + (1 << 22))
        x[i:i + (1 << 22)] = (rng.standard_normal(1 << 22) + np.cos(2 * np.pi * 0.1 * t)).astype(np.float32)
    p = dsp.welch_pgram(x, nseg, hop, window=dsp.hanning).power
    assert p.shape == (2049,) and p.dtype == np.float32
    w = ow.hanning(nseg)
    k = (n - nseg) // hop + 1
    # sum_k P[k] * (fs/nfft) == mean_seg sum |w x|^2 / norm2   (two-sided; one-sided doubles the interior bins)
    x64 = x.astype(np.float64)
    w2a, w2b = w[:hop] ** 2, w[hop:] ** 2
    blocks = (x64[: (k + 1) * hop] ** 2).reshape(k + 1, hop)
    seg_energy = blocks[:-1] @ w2a + blocks[1:] @ w2b
    lhs = p.astype(np.float64).sum() / nseg
    rhs = seg_energy.mean() / np.sum(w ** 2)
    assert abs(lhs - rhs) / rhs < TOL32
    # the tone bin via a direct DFT of every segment at that bin (bin 410 ~ 0.1 * 4096 = 409.6 -> check 409, 410)
    for kb in (409, 410, 7):
        e = np.exp(-2j * np.pi * kb * np.arange(nseg) / nseg) * w
        ea, eb = e[:hop], e[hop:]
        xb = x64[: (k + 1) * hop].reshape(k + 1, hop)
        X = xb[:-1] @ ea + xb[1:] @ eb
        ref = 2 * np.mean(np.abs(X) ** 2) / np.sum(w ** 2)
        assert abs(p[kb] - ref) / ref < TOL32


def test_spectrogram_config4_batched():
    # BASELINE config 4 shape (channels x 2^18): batched call == per-channel calls == oracle
    rng = np.random.default_rng(1004)
    nchan, length = 8, 1 << 18
    t = np.arange(length)
    x = np.stack([np.cos(2 * np.pi * (0.05 + 0.1 * c / nchan) * t * (1 + t / length) / 2) + 0.1 * rng.standard_normal(length)
                  for c in range(nchan)], axis=1).astype(np.float32)
    sp = dsp.spectrogram(x, 1024, 768)
    assert sp.power.shape == (513, (length - 1024) // 256 + 1, nchan) and sp.power.dtype == np.float32
    for c in (0, 3, 7):
        one = dsp.spectrogram(x[:, c], 1024, 768)
        assert np.array_equal(one.power, sp.power[:, :, c])
        truth, _, _ = op.spectrogram(x[:, c], 1024, 768, f64=True)
        assert relerr(one.power, truth) < TOL32
    sph = dsp.spectrogram(x[:, 1], 1024, 768, window=dsp.hanning)
    assert relerr(sph.power, op.spectrogram(x[:, 1], 1024, 768, window=ow.hanning, f64=True)[0]) < TOL32


# =============================================================================== resample

@pytest.mark.parametrize("rate", ["1/2", "2/1", "3/2", "2/3"])
def test_resample_matlab_goldens(goldens, rate):
    # test/resample.jl:8-24
    r = Fraction(rate)
    key = f"{r.numerator}_{r.denominator}"
    x, h, y = goldens["resample_x"], goldens[f"resample_taps_{key}"], goldens[f"resample_y_{key}"]
    yj = dsp.resample(x, r, h)
    assert yj.shape == y.shape and approx(yj, y)
    assert relerr(yj, of.resample_literal(x, r, h)) < TOL64
    assert approx(dsp.resample(x, r), y, rtol=1e-3)
    assert np.array_equal(dsp.resample(x, r), dsp.resample(x, r, dsp.resample_filter(r)))   # test/resample.jl:26-32


def test_resample_exact_tiny_and_dims():
    # test/filt_stream.jl:366-367; test/resample.jl:26-72 (dims)
    h = np.array([0, 0, 1, 0, 0, 0.])
    assert np.array_equal(dsp.resample(np.array([1., 2.]), 3, h), [1, 0, 0, 2, 0, 0])
    assert np.array_equal(dsp.resample(np.array([1., 2.]), "3//2", h), [1, 0, 0])
    m = randn(121 * 7, np.float64).reshape(121, 7)
    r = dsp.resample(m, Fraction(3, 2), dims=0)
    for c in range(7):
        assert np.array_equal(r[:, c], dsp.resample(m[:, c], Fraction(3, 2)))
    r1 = dsp.resample(m.T.copy(), Fraction(3, 2), dims=1)
    assert np.array_equal(r1, r.T)


@pytest.mark.parametrize("th", [np.float32, np.float64])
@pytest.mark.parametrize("tx", [np.float32, np.float64, np.complex64, np.complex128])
def test_resample_grid_vs_reference_loops(th, tx):
    # test/filt_stream.jl:231-281, 338-364: interp x decim x Th x Tx against the stateful reference loops
    for interp in (1, 5, 14, 23):
        for dec in (1, 9, 17, 21):
            if interp == dec:
                continue
            r = Fraction(interp, dec)
            h = randn(56, th)
            x = randn(401, tx)
            y = dsp.resample(x, r, h)
            ref = of.resample_literal(x, r, h)
            assert y.dtype == np.result_type(th, tx) and y.shape == ref.shape, (interp, dec)
            truth = of.resample(x, r, h, f64=True)
            assert relerr(y, truth) < tol(y.dtype), (interp, dec)
            assert relerr(ref, truth) < 50 * tol(y.dtype)


def test_resample_config5_scaled():
    # BASELINE config 5 shape at 2^20: 3//2 on ComplexF32 with the default taps (Float64 -> ComplexF64 out,
    # Appendix B) and with Float32 taps (ComplexF32 out)
    x = randn(1 << 20, np.complex64)
    h = dsp.resample_filter(Fraction(3, 2))
    assert h.size == 111
    y64 = dsp.resample(x, Fraction(3, 2))
    assert y64.dtype == np.complex128 and y64.size == 3 * (1 << 19)
    assert relerr(y64, of.resample(x, Fraction(3, 2), h)) < TOL64
    y32 = dsp.resample(x, Fraction(3, 2), h.astype(np.float32))
    assert y32.dtype == np.complex64
    assert relerr(y32, of.resample(x, Fraction(3, 2), h.astype(np.float32), f64=True)) < TOL32


# =============================================================================== FIRFilter streaming / arraysplit / fftshift

@pytest.mark.parametrize("tx", [np.float32, np.complex128])
def test_firfilter_streaming_matches_reference_loops(tx):
    # test/filt_stream.jl:231-281, 338-364: stateless, two-chunk and many-small-chunk filtering all equal the
    # reference's stateful loops (single-rate, interpolation, decimation, rational)
    for interp in (1, 5, 14):
        for dec in (1, 9, 17):
            r = Fraction(interp, dec)
            h = randn(56, np.float64)
            x = randn(1201, tx)
            ref = of.FIRFilterState(h, r).filt(x)
            y1 = dsp.FIRFilter(h, r).filt(x)
            assert y1.shape == ref.shape and relerr(y1, ref) < 50 * tol(y1.dtype), (interp, dec)
            assert np.array_equal(dsp.filt(h, x, r), y1)                       # filt(h, x, ratio), stream_filt.jl:663-666
            f2 = dsp.FIRFilter(h, r)
            cut = 433
            y2 = np.concatenate([f2.filt(x[:cut]), f2.filt(x[cut:])])
            assert y2.shape == ref.shape and relerr(y2, ref) < 50 * tol(y1.dtype), (interp, dec)
            f3, parts, pos = dsp.FIRFilter(h, r), [], 0
            for step in (1, 2, 3, 1, 40, 1, 7, 300, 1, 1, 844):
                parts.append(f3.filt(x[pos:pos + step]))
                pos += step
            assert pos == x.size
            y3 = np.concatenate(parts)
            assert y3.shape == ref.shape and relerr(y3, ref) < 50 * tol(y1.dtype), (interp, dec)
            ro = of.FIRFilterState(h, r)
            ro.filt(x)
            assert (f3.phi_idx, f3.input_deficit) == (ro.phi_idx, ro.input_deficit), (interp, dec)
            f3.reset()
            assert np.array_equal(f3.filt(x), y1)


def test_arraysplit_and_fftshift():
    # test/periodograms.jl:393-402 (#124) and the docstring examples src/periodograms.jl:96-113
    q = dsp.arraysplit(np.ones(1000), 100, 10)
    assert q.shape == (11, 100) and np.array_equal(q.mean(axis=1), np.ones(11))
    a = dsp.arraysplit(np.array([0.1, 0.2, 0.3, 0.4, 0.5]), 3, 2, 8)
    assert a.shape == (3, 8) and np.array_equal(a[2, :3], [0.3, 0.4, 0.5]) and not a[:, 3:].any()
    b = dsp.arraysplit(np.array([0.1, 0.2, 0.3, 0.4, 0.5]), 3, 1, 3, np.array([1, 2, 1]))
    assert np.allclose(b, [[0.1, 0.4, 0.3], [0.3, 0.8, 0.5]])
    x = randn(5000, np.float32)
    w = dsp.hanning(512)
    assert np.array_equal(dsp.arraysplit(x, 512, 384, 1024, w), op.arraysplit(x, 512, 384, 1024, w)) or \
        relerr(dsp.arraysplit(x, 512, 384, 1024, w), op.arraysplit(x, 512, 384, 1024, w)) < 1e-7
    with pytest.raises(dsp.DomainError):
        dsp.arraysplit(np.ones(10), 4, 4)
    # more than 65535 segments: several launches of up to 65535 segments each, on a cuFFT-size and a fused plan.  The
    # window is exact in Float32, so the oracle's Float64 product rounded once is the kernel's product.
    x = randn(600000, np.float32)
    for n, noverlap, nfft in ((16, 8, None), (64, 56, 256)):
        w = dsp.hanning(n).astype(np.float32).astype(np.float64)
        q = dsp.arraysplit(x, n, noverlap, nfft, w)
        assert q.shape[0] > 65535 and np.array_equal(q, op.arraysplit(x, n, noverlap, nfft, w, f64=False))
    # test/periodograms.jl:239-248
    p = dsp.periodogram(DATA)
    ps = dsp.fftshift(p)
    assert np.array_equal(p.power, ps.power) and np.allclose(p.freq, ps.freq)
    p2 = dsp.periodogram(DATA, onesided=False)
    p2s = dsp.fftshift(p2)
    assert np.array_equal(np.fft.fftshift(p2.power), p2s.power) and np.array_equal(np.fft.fftshift(p2.freq), p2s.freq)
    assert np.array_equal(dsp.fftshift(p2s).power, p2s.power)


def test_device_array_pipeline():
    # device-resident pipeline (the analogue of handing CuArrays to the Julia glue): identical results to the host path
    u = randn(300000, np.complex64)
    v = randn(513, np.complex64)
    ud = dsp.to_device(u)
    yd = dsp.conv(ud, v, algorithm="fft_overlapsave")
    y = dsp.conv(u, v, algorithm="fft_overlapsave")
    assert isinstance(yd, dsp.DeviceArray) and yd.shape == y.shape
    assert np.array_equal(yd.to_host(), y)
    p = dsp.welch_pgram(yd[:u.size], 1024, 512, window=dsp.hanning)
    assert np.array_equal(p.power, dsp.welch_pgram(y[:u.size], 1024, 512, window=dsp.hanning).power)
    cfg = dsp.WelchConfig(u.size, np.complex64, n=1024, noverlap=512, window=dsp.hanning)
    assert np.array_equal(dsp.welch_pgram(yd[:u.size], cfg).power, p.power)
    xr = randn(200000, np.float32)
    b = randn(300, np.float32)
    xd = dsp.to_device(xr)
    assert np.array_equal(dsp.fftfilt(b, xd).to_host(), dsp.fftfilt(b, xr))
    sp = dsp.spectrogram(xd, 1024, 768)
    assert np.array_equal(sp.power.to_host(), dsp.spectrogram(xr, 1024, 768).power)
    z = dsp.resample(dsp.to_device(u[:100001]), Fraction(3, 2))
    assert np.array_equal(z.to_host(), dsp.resample(u[:100001], Fraction(3, 2)))
    del ud, yd, xd, z
    dsp.device.empty_cache()


# =============================================================================== thin clients (SURVEY.md 8f rank 3)

def test_xcorr_reference_cases():
    # test/dsp.jl:317-345
    a, b = [1, 2, 3], [4, 5]
    exp = [5, 14, 23, 12]
    assert np.array_equal(dsp.xcorr([1, 2], [3, 4]), [4, 11, 6])
    assert np.array_equal(dsp.xcorr(a, b), exp)
    assert np.array_equal(dsp.xcorr(a, b, padmode="longest"), [0, 5, 14, 23, 12])
    assert np.array_equal(dsp.xcorr(a, b, padmode="none"), exp)
    assert np.array_equal(dsp.xcorr([1, 2], [3, 4, 5]), [5, 14, 11, 6])
    assert np.array_equal(dsp.xcorr([1, 2], [3, 4, 5], padmode="longest"), [5, 14, 11, 6, 0])
    assert np.array_equal(dsp.xcorr([1.0j], [1.0j]), [1])
    assert approx(dsp.xcorr(np.array(a) * 1.0j, np.array(b, dtype=complex)), np.array(exp) * 1j)
    assert approx(dsp.xcorr(np.array(a, dtype=complex), np.array(b) * 1.0j), -np.array(exp) * 1j)
    assert approx(dsp.xcorr(np.array(a) * 1.0j, np.array(b) * 1.0j), np.array(exp, dtype=complex))
    assert np.array_equal(dsp.xcorr([1, 2, 3]), [3, 8, 14, 8, 3])
    assert approx(dsp.xcorr([1., 2, 3], scaling="biased"), np.array([3, 8, 14, 8, 3]) / 3)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.xcorr(a, b, scaling="biased")
    with pytest.raises(dsp.ArgumentError):
        dsp.xcorr(a, b, padmode="bogus")
    u, v = randn(3000, np.complex64), randn(700, np.complex64)       # large enough for the FFT path
    ref = np.correlate(u.astype(np.complex128), v.astype(np.complex128), mode="full")
    assert relerr(dsp.xcorr(u, v), ref) < TOL32


def test_finddelay_shiftsignal_alignsignals():
    # test/util.jl:125-170
    x = randn(200, np.float64)
    d = 17
    xd = np.concatenate([np.zeros(d), x])
    assert dsp.finddelay(xd, x) == d and dsp.finddelay(xd, -x) == d
    assert dsp.finddelay(x, xd) == -d and dsp.finddelay(-x, xd) == -d
    assert np.array_equal(dsp.shiftsignal(x, d), np.concatenate([np.zeros(d), x[:-d]]))
    assert np.array_equal(dsp.shiftsignal(x, -d), np.concatenate([x[d:], np.zeros(d)]))
    y, s = dsp.alignsignals(xd, x)
    assert s == d and np.array_equal(y, np.concatenate([x, np.zeros(d)]))
    y, s = dsp.alignsignals(x, xd)
    assert s == -d and np.array_equal(y, np.concatenate([np.zeros(d), x[:-d]]))
    assert dsp.alignsignals([0, 0, 1, 2, 3], [1, 2, 3])[1] == 2
    with pytest.raises(dsp.DomainError):
        dsp.shiftsignal([1], -2)


@pytest.mark.parametrize("rate", [0.7312, 1.2957, 2.618, 1 / 55.55])
@pytest.mark.parametrize("dt", [np.float32, np.float64, np.complex64, np.complex128])
def test_arbitrary_rate_filter_vs_literal_loop(rate, dt):
    # FIRFilter{FIRArbitrary}: test/filt_stream.jl:288-353 -- stateless, stateful and chunked filtering
    nphi = 32
    h = dsp.resample_filter(rate, nphi)
    x = randn(700, dt)
    want = of.FIRArbitraryState(h, rate, nphi).filt(x)
    # The comparison target is the reference's LITERAL loop, whose Float64 phase accumulator is a running sum (acc += delta,
    # wrapped every output): its rounding random-walks by ~sqrt(j) * Nphi * eps and the interpolated output moves with the
    # phase, while the kernel evaluates acc0 + j * delta per output in double-double (closer to exact arithmetic, DESIGN.md
    # section 7).  The two therefore agree to ~1e-11 (Float64) / ~2e-6 (Float32 outputs), not to the 1e-12 / 1e-6 the
    # kernels reach against an exact-phase oracle; rate 1/55.55 has the most phase steps per output.
    tol = 2e-6 if np.dtype(dt) in (np.dtype(np.float32), np.dtype(np.complex64)) else 1e-11
    got = dsp.filt_multirate(h, x, rate, nphi)
    assert got.dtype == want.dtype and got.size == want.size
    assert relerr(got, want) < tol
    sf = dsp.FIRFilter(h, rate, nphi)
    assert relerr(sf.filt(x), want) < tol
    sf.reset()
    so = of.FIRArbitraryState(h, rate, nphi)
    pos, pieces = 0, []
    for step in (1, 1, 3, 64, 0, 200, 5, 426):
        chunk = x[pos:pos + step]
        pieces.append(sf.filt(chunk))
        ref = so.filt(chunk)
        assert pieces[-1].size == ref.size and sf.input_deficit == so.input_deficit
        assert abs(sf.phi_accumulator - so.acc) < 1e-9
        pos += step
    assert pos == x.size and relerr(np.concatenate(pieces), want) < tol
    # Float32 taps stay in single precision with Float32 signals (promote_type)
    if np.dtype(dt) in (np.dtype(np.float32), np.dtype(np.complex64)):
        h32 = h.astype(np.float32)
        w32 = of.FIRArbitraryState(h32, rate, nphi).filt(x)
        g32 = dsp.filt_multirate(h32, x, rate, nphi)
        assert g32.dtype == w32.dtype == np.dtype(dt) and relerr(g32, w32) < 5e-6      # Float32 taps AND literal-loop phases


def test_arbitrary_rate_resample():
    # test/resample.jl:38-54, 99-107
    assert dsp.resample(np.sin(np.arange(1.0, 35547.0)), 1 / 55.55).size == 640
    x = np.random.default_rng(0).standard_normal(1822)
    y = dsp.resample(x, 0.9802414928649835)
    assert y.size == 1786 and relerr(y, of.resample_arb_literal(x, 0.9802414928649835)) < 1e-10
    assert np.array_equal(dsp.resample(np.zeros(1000), 0.012), np.zeros(12))
    assert dsp.resample(np.arange(1, 16_367_000 * 2 + 1), 10_000_000 / 16_367_000).size == 20_000_000
    # a float rate that is an exact ratio agrees with the rational resampler to the quality of the default taps
    t = np.arange(2000) / 100.0
    sig = np.sin(2 * np.pi * 1.3 * t)
    ya, yr = dsp.resample(sig, 1.5), dsp.resample(sig, Fraction(3, 2))
    assert ya.size == yr.size and np.abs(ya[50:-50] - yr[50:-50]).max() < 2e-3
    X = np.stack([sig, 2 * sig], axis=1)
    Y = dsp.resample(X, 1.5, dims=0)
    assert Y.shape == (3000, 2) and np.array_equal(Y[:, 0], ya) and relerr(Y[:, 1], 2 * ya) < 1e-12
    assert np.array_equal(dsp.resample(X.T, 1.5, dims=1), Y.T)
    with pytest.raises(dsp.DomainError):
        dsp.resample(sig, -0.5)


def test_periodogram_2d_reference_cases(goldens):
    # test/periodograms.jl:270-330, 391
    x = goldens["per2dx"]
    assert relerr(dsp.periodogram(x, fs=1, radialsum=True).power, goldens["per2dsum"]) < 1e-10
    assert relerr(dsp.periodogram(x, fs=1, radialavg=True).power, goldens["per2dmean"]) < 1e-10
    p = dsp.periodogram(x, fs=1)
    assert isinstance(p, dsp.Periodogram2) and relerr(p.power, np.abs(np.fft.fft2(x)) ** 2 / x.size) < TOL64
    pads = (x.shape[0] + 4, x.shape[0] + 7)
    xp = np.zeros(pads)
    xp[:x.shape[0], :x.shape[1]] = x
    assert relerr(dsp.periodogram(x, fs=1, nfft=pads).power, np.abs(np.fft.fft2(xp)) ** 2 / x.size) < TOL64
    assert np.allclose(dsp.periodogram(x, fs=3.3, radialsum=True).freq, dsp.periodogram(x[0, :], fs=3.3).freq)
    f1, f2 = dsp.periodogram(x, fs=3.3).freq
    f1d = dsp.periodogram(x[0, :], fs=3.3, onesided=False).freq
    assert np.allclose(f1, f1d) and np.allclose(f2, f1d)
    ps = dsp.fftshift(p)
    assert np.array_equal(ps.power, np.fft.fftshift(p.power)) and np.array_equal(ps.freq1, np.fft.fftshift(p.freq1))
    # non-square signal that is sparse in FFT space (test "radial")
    n1, n2, nf = 52, 46, (21, 6)
    F1, F2 = np.fft.fftfreq(n1), np.fft.fftfreq(n2)
    X = np.zeros((n1, n2), dtype=complex)
    X[nf] = 1 + 2j
    X[(-nf[0]) % n1, (-nf[1]) % n2] = 1 - 2j
    y = np.real(np.fft.ifft2(X))
    fwn = int(np.rint(np.hypot(F1[nf[0]], F2[nf[1]]) * n2))
    pe = np.zeros((n2 >> 1) + 1)
    pe[fwn] = 2 * abs(X[nf]) ** 2 / n1 / n2
    P = dsp.periodogram(y, nfft=(n1, n2), radialsum=True)
    assert np.allclose(P.power, pe, atol=1e-12) and abs(P.freq[fwn] - fwn / n2) < 1e-15
    # both precisions against the literal restatement, with padding and a non-square transform
    for dt, tol in ((np.float64, 1e-11), (np.float32, 2e-6)):        # against the literal accumulator loop, see above
        z = randn((37, 50), dt)
        for kw in ({}, {"radialsum": True}, {"radialavg": True}, {"nfft": (64, 50), "radialavg": True}, {"nfft": (40, 81)}):
            got = dsp.periodogram(z, fs=2.5, **kw)
            want = op.periodogram2(z, fs=2.5, **kw)
            assert got.power.dtype == want[0].dtype and relerr(got.power, want[0]) < tol
    assert np.allclose(dsp.periodogram(np.array([[1, 3], [0, 1]]), radialavg=True).power, [6.25, 1.5833333333333333])
    with pytest.raises(dsp.ArgumentError):
        dsp.periodogram(np.array([[1, 2], [3, 4]]), radialsum=True, radialavg=True)
    with pytest.raises(dsp.ArgumentError):
        dsp.periodogram(np.ones((4, 4)), nfft=(3, 4))


def test_conv_2d_reference_cases():
    # test/dsp.jl:130-224
    a = np.array([[1, 2, 1], [2, 3, 1], [1, 2, 1]])
    b = np.array([[3, 2], [0, 1]])
    expectation = np.array([[3, 8, 7, 2], [6, 14, 11, 3], [3, 10, 10, 3], [0, 1, 2, 1]])
    im_expectation = np.array([[3, 5, 5, 2], [3, 6, 6, 3], [3, 6, 6, 3], [0, 1, 1, 1]])
    assert np.array_equal(dsp.conv(a, b), expectation) and dsp.conv(a, b).dtype.kind == "i"
    assert np.array_equal(dsp.conv(a.astype(np.int32), b), expectation)
    fa, fb = a.astype(np.float64), b.astype(np.float64)
    assert np.array_equal(dsp.conv(fa, fb), expectation)
    assert np.array_equal(dsp.conv(fa + 1j, fb + 0j), expectation + 1j * im_expectation)
    assert relerr(dsp.conv(fa, b), expectation) < TOL64 and relerr(dsp.conv(fb, a), expectation) < TOL64
    assert relerr(dsp.conv(a.astype(np.float32), b), expectation) < TOL64        # Float32 x Int -> Float64
    u, v = randn((10, 20), np.float64), randn((10, 10), np.float64)
    ref = od.conv_td_nd(u, v)
    for alg in ("direct", "fft_simple", "fft_overlapsave", "fft", "fast", "auto"):
        assert relerr(dsp.conv(u, v, algorithm=alg), ref) < TOL64
    with pytest.raises(dsp.ArgumentError):
        dsp.conv(u, v, algorithm="quantum")
    from scipy.signal import convolve
    for (M1, M2) in ((10, 20), (190, 200)):
        for (N1, N2) in ((20, 10), (210, 200)):
            for dt, tol in ((np.float64, TOL64), (np.complex128, TOL64), (np.float32, TOL32), (np.complex64, TOL32)):
                u, v = randn((M1, M2), dt), randn((N1, N2), dt)
                wide = np.complex128 if np.dtype(dt).kind == "c" else np.float64
                ref = convolve(u.astype(wide), v.astype(wide), method="fft" if M1 > 100 else "direct")
                got = dsp.conv(u, v, algorithm="fft_simple")
                assert got.dtype == np.dtype(dt) and got.shape == (M1 + N1 - 1, M2 + N2 - 1) and relerr(got, ref) < tol
                assert relerr(got, od.conv_kern_fft_nd(u, v, f64=True)) < tol
                if M1 * M2 * N1 * N2 < 1 << 22:
                    assert relerr(dsp.conv(u, v, algorithm="direct"), ref) < tol
    # separable kernel: conv(u, v', A)
    su, sv = np.array([1, 2, 3, 2, 1]), np.array([6, 7, 3, 2])
    A = np.arange(1, 29).reshape(4, 7)
    exp = np.array([[6, 19, 35, 53, 71, 89, 107, 77, 33, 14], [60, 148, 217, 285, 339, 393, 447, 315, 134, 56],
                    [204, 478, 658, 822, 930, 1038, 1146, 798, 338, 140], [468, 1062, 1400, 1684, 1828, 1972, 2116, 1456, 614, 252],
                    [636, 1426, 1848, 2188, 2332, 2476, 2620, 1792, 754, 308], [624, 1388, 1778, 2082, 2190, 2298, 2406, 1638, 688, 280],
                    [354, 785, 1001, 1167, 1221, 1275, 1329, 903, 379, 154], [132, 292, 371, 431, 449, 467, 485, 329, 138, 56]])
    assert relerr(dsp.conv(su.astype(np.float64), sv.astype(np.float64), A.astype(np.float64)), exp) < TOL64


def test_conv_3d_and_mixed_rank():
    # test/dsp.jl:225-262 (conv-ND) + rank promotion, src/dspbase.jl:784-792
    from scipy.signal import convolve
    for dt, tol in ((np.float64, TOL64), (np.complex64, TOL32)):
        u, v = randn((7, 9, 5), dt), randn((4, 3, 6), dt)
        wide = np.complex128 if np.dtype(dt).kind == "c" else np.float64
        ref = convolve(u.astype(wide), v.astype(wide), method="direct")
        for alg in ("direct", "fft_simple", "fft_overlapsave", "auto"):
            got = dsp.conv(u, v, algorithm=alg)
            assert got.shape == ref.shape and relerr(got, ref) < tol
        w = randn(6, dt)
        assert relerr(dsp.conv(u, w), convolve(u.astype(wide), w.astype(wide).reshape(6, 1, 1))) < tol
        assert relerr(dsp.conv(w, u[:, :, 0]), convolve(w.astype(wide).reshape(6, 1), u[:, :, 0].astype(wide))) < tol
    big_u, big_v = randn((64, 48, 40), np.float32), randn((9, 7, 5), np.float32)
    assert relerr(dsp.conv(big_u, big_v), convolve(big_u.astype(np.float64), big_v.astype(np.float64), method="fft")) < TOL32
    assert dsp.conv(np.zeros((0, 3)), np.ones((2, 2))).shape == (1, 4)
    ints = np.arange(24).reshape(2, 3, 4)
    assert np.array_equal(dsp.conv(ints, ints), od.conv_td_nd(ints, ints))
    a = np.arange(1, 28).reshape((3, 3, 3), order="F")                        # test/dsp.jl:232-252
    exp = np.array([1, 3, 5, 3, 5, 12, 16, 9, 11, 24, 28, 15, 7, 15, 17, 9, 11, 24, 28, 15, 28, 60, 68, 36, 40, 84, 92, 48, 23, 48, 52, 27,
                    29, 60, 64, 33, 64, 132, 140, 72, 76, 156, 164, 84, 41, 84, 88, 45, 19, 39, 41, 21, 41, 84, 88, 45, 47, 96, 100, 51,
                    25, 51, 53, 27]).reshape((4, 4, 4), order="F")
    assert np.array_equal(dsp.conv(a, np.ones((2, 2, 2), dtype=np.int64)), exp)
    layers = np.stack([np.full((3, 3), n) for n in range(1, 7)], axis=2)      # promote dims to largest, test/dsp.jl:259-262
    k2 = np.ones((2, 2), dtype=np.int64)
    assert np.array_equal(dsp.conv(layers, k2), od.conv_td_nd(layers, k2)) and dsp.conv(layers, k2).shape == (4, 4, 6)


def test_conv_nd_overlap_save_blocks():
    # test/dsp.jl:270-313 ("Overlap-Save"): unsafe_conv_kern_os! with nffts = optimalfftfiltlength(nsmall, nlarge) in every
    # dimension against _conv_kern_fft!, N = 1, 2, 3; here: the N-D blocked path of the library (batched cuFFT blocks)
    # against the restated block loop (small cases, same nffts) and against one big transform pair in Float64
    from dspb200 import _lib

    def run_os(u, v, nffts):
        out = np.empty(tuple(a + b - 1 for a, b in zip(u.shape, v.shape)), dtype=u.dtype, order="F")
        _lib.conv_nd(np.asfortranarray(u), np.asfortranarray(v), nffts, out, overlapsave=True)
        return out

    nlarge = 128
    for nd in (1, 2, 3):
        for dt, tl in ((np.float32, TOL32), (np.float64, TOL64), (np.complex128, TOL64)):
            for nsmall in (12, 128):
                if nd == 3 and nsmall == 128 and dt is not np.float32:
                    continue                                        # 255^3 outputs: one precision is enough for the suite's time
                nfft = dsp.optimalfftfiltlength(nsmall, nlarge)
                u, v = randn((nlarge,) * nd, dt), randn((nsmall,) * nd, dt)
                got = run_os(u, v, (nfft,) * nd)
                want = od.conv_kern_fft_nd(u, v, f64=True)
                assert got.dtype == np.dtype(dt) and got.shape == want.shape and relerr(got, want) < tl, (nd, dt, nsmall)
                assert relerr(dsp.conv(u, v, algorithm="fft_overlapsave"), want) < tl
    # adversarial (nsmall, nfft) of the reference: output smaller than a block's valid region; sout divisible / not divisible
    # by the block size; three padded blocks (25, 4, 16)
    for nl, ns, nfft in ((128, 12, 256), (128, 13, 32), (128, 12, 32), (25, 4, 16)):
        for nd in (1, 2):
            u, v = randn((nl,) * nd, np.float64), randn((ns,) * nd, np.float64)
            got = run_os(u, v, (nfft,) * nd)
            assert relerr(got, od.conv_kern_os_nd(u, v, (nfft,) * nd)) < TOL64
            assert relerr(got, od.conv_td_nd(u, v)) < TOL64
    # different transform per dimension, v longer than u in one dimension, singleton dimensions
    for su, sv, nf, dt, tl in (((40, 37), (5, 9), (16, 32), np.complex64, TOL32), ((20, 9, 17), (3, 4, 2), (8, 8, 16), np.float32, TOL32),
                               ((4, 7, 1), (3, 3, 3), (8, 8, 4), np.float64, TOL64), ((33, 1, 29), (7, 1, 3), (16, 1, 8), np.float64, TOL64)):
        u, v = randn(su, dt), randn(sv, dt)
        assert relerr(run_os(u, v, nf), od.conv_kern_os_nd(u, v, nf, f64=True)) < tl
    dsp.conv(np.zeros((4, 7, 1)), np.zeros((3, 3, 3)))                        # "Should not bug", test/dsp.jl:309
    # several batches and a partial last batch: 9 x 8 blocks of 32 x 32 Float64 samples, five blocks per batch
    u, v = randn((200, 150), np.float64), randn((9, 11), np.float64)
    whole = run_os(u, v, (32, 32))
    _lib.conv_nd_os_set_budget(5 * (32 * 32 * 8 + 17 * 32 * 16))
    try:
        pieces = run_os(u, v, (32, 32))
    finally:
        _lib.conv_nd_os_set_budget(1 << 30)
    assert np.array_equal(whole, pieces) and relerr(whole, od.conv_td_nd(u, v)) < TOL64
    with pytest.raises(dsp.DSPB200Error):
        run_os(u, v, (8, 32))                                                   # nffts below size(v)


def test_nd_conv_periodogram2_and_multitaper_device_resident():
    # the *_dev twins of the widened rows: device-resident inputs give device-resident results equal to the host-pointer calls
    u, v = randn((96, 70), np.float32), randn((9, 5), np.float32)
    for alg in ("direct", "fft_simple", "fft_overlapsave"):
        d = dsp.conv(dsp.to_device(u), dsp.to_device(v), algorithm=alg)
        assert isinstance(d, dsp.DeviceArray) and d.shape == (104, 74)
        assert np.array_equal(dsp.to_host(d), dsp.conv(u, v, algorithm=alg))
    d = dsp.conv(dsp.to_device(v), u, algorithm="fft_overlapsave")              # smaller array first, mixed host / device
    assert np.array_equal(dsp.to_host(d), dsp.conv(v, u, algorithm="fft_overlapsave"))
    u3, v3 = randn((30, 20, 10), np.complex128), randn((4, 3, 2), np.complex128)
    assert np.array_equal(dsp.to_host(dsp.conv(dsp.to_device(u3), dsp.to_device(v3), algorithm="fft_simple")),
                          dsp.conv(u3, v3, algorithm="fft_simple"))
    z = randn((37, 50), np.float64)
    for kw in ({}, {"radialsum": True}, {"nfft": (64, 50), "radialavg": True}):
        got = dsp.periodogram(dsp.to_device(z), fs=2.5, **kw)
        want = dsp.periodogram(z, fs=2.5, **kw)
        assert isinstance(got.power, dsp.DeviceArray)
        if kw:                                                      # radial rings: Float64 atomics, summation order not fixed
            assert relerr(dsp.to_host(got.power), want.power) < TOL64
        else:
            assert np.array_equal(dsp.to_host(got.power), want.power)
    x = randn(3000, np.float32)
    assert np.array_equal(dsp.periodogram(dsp.to_device(x), fs=3, window=dsp.hanning).power, dsp.periodogram(x, fs=3, window=dsp.hanning).power)
    assert np.array_equal(dsp.to_host(dsp.mt_pgram(dsp.to_device(x), fs=10, nw=3).power), dsp.mt_pgram(x, fs=10, nw=3).power)
    for n, nov in ((1000, 500), (300, 100)):                                       # nfft = 1024 and 512
        a = dsp.mt_spectrogram(dsp.to_device(x), n, nov, nw=3)
        b = dsp.mt_spectrogram(x, n, nov, nw=3)
        assert isinstance(a.power, dsp.DeviceArray) and np.array_equal(dsp.to_host(a.power), b.power)
    sig = randn((4, 600), np.float64)
    for coh in (False, True):
        fn = dsp.mt_coherence if coh else dsp.mt_cross_power_spectra
        a = fn(dsp.to_device(sig), fs=1, demean=True, freq_range=(0.1, 0.3), nw=3)
        b = fn(sig, fs=1, demean=True, freq_range=(0.1, 0.3), nw=3)
        got = dsp.to_host(a.coherence if coh else a.power)
        assert np.array_equal(got, b.coherence if coh else b.power)


def _mt_cross_case(goldens):
    fs, n = 1000.0, 1024
    t = np.arange(n) / fs
    sin_1 = np.sin(2 * np.pi * 12.0 * t)
    sin_2 = np.sin(np.pi * (2 * 12.0 * t + 1))
    return fs, n, sin_1, sin_2


def test_mt_cross_power_spectra_mne_golden(goldens):
    # test/multitaper.jl:277-330
    fs, n, sin_1, sin_2 = _mt_cross_case(goldens)
    signal = np.stack([sin_1, sin_2])
    ref = (goldens["csd_mt_values_re"] + 1j * goldens["csd_mt_values_im"]).reshape((512, 2, 2)).transpose(2, 1, 0)
    mt_config = dsp.dpss_config(np.float64, n, fs=fs, keep_only_large_evals=True, weight_by_evals=True)
    assert mt_config.ntapers == 7
    config = dsp.MTCrossSpectraConfig(2, mt_config, demean=True)
    result = dsp.mt_cross_power_spectra(signal, config)
    assert result.power.dtype == np.complex128 and result.power.shape == (2, 2, 513)
    assert np.allclose(result.freq[1:], goldens["csd_mt_frequencies"])
    assert relerr(result.power[:, :, 1:], ref) < TOL64
    # Float32 configuration, Float64 and Float32 input
    mt32 = dsp.dpss_config(np.float32, n, fs=fs, keep_only_large_evals=True, weight_by_evals=True)
    c32 = dsp.MTCrossSpectraConfig(2, mt32, demean=True)
    for sig in (signal, signal.astype(np.float32)):
        r32 = dsp.mt_cross_power_spectra(sig, c32)
        assert r32.power.dtype == np.complex64 and relerr(r32.power[:, :, 1:], ref) < TOL32
    with pytest.raises(dsp.DimensionMismatch):
        dsp.mt_cross_power_spectra(np.vstack([signal, signal]), config)
    with pytest.raises(dsp.ArgumentError):
        dsp.MTCrossSpectraConfig(2, dsp.MTConfig(np.complex64, n))


def test_mt_coherence_reference_cases(goldens):
    # test/multitaper.jl:96-275
    fs, n, sin_1, sin_2 = _mt_cross_case(goldens)
    noise = goldens["mt_noise"]
    mt_config = dsp.dpss_config(np.float64, n, fs=fs, keep_only_large_evals=True, weight_by_evals=True)
    config = dsp.MTCrossSpectraConfig(2, mt_config, freq_range=(10, 15), demean=True)
    c = dsp.mt_coherence(np.stack([sin_1, sin_1 + 3 * noise]), config)
    assert np.all((c.freq >= 10) & (c.freq <= 15)) and c.coherence.shape == (2, 2, c.freq.size)
    assert abs(c.coherence.mean(axis=2)[1, 0] - 0.982356762670818) < 1e-10        # MNE-python value
    assert np.array_equal(c.coherence, np.transpose(c.coherence, (1, 0, 2)))
    assert np.all(c.coherence[0, 0] == 1) and np.all(c.coherence[1, 1] == 1)
    avg = lambda sig, **kw: dsp.mt_coherence(sig, fs=fs, freq_range=(10, 15), **kw).coherence.mean(axis=2)
    same = avg(np.stack([sin_1, sin_1]), demean=True)[1, 0]
    shift = avg(np.stack([sin_1, sin_2]))[1, 0]
    assert abs(same - 1) < 1e-5 and abs(shift - 1) < 1e-5
    rn = np.random.default_rng(11).uniform(-1, 1, n)
    diff = avg(np.stack([sin_1, rn]))[1, 0]
    less = avg(np.stack([sin_1, sin_1 + rn]))[1, 0]
    more = avg(np.stack([sin_1, sin_1 + 3 * rn]))[1, 0]
    assert diff < 0.8 and less < same and more < less and diff < more
    several = avg(np.stack([sin_1, sin_2, rn]))
    assert several.shape == (3, 3) and abs(several[1, 0] - shift) < 1e-9 and abs(several[2, 0] - diff) < 1e-9
    # against the oracle on a random multichannel case, all dtypes, with and without a frequency range
    x = randn((5, 600), np.float64)
    for dt, tol in ((np.float64, TOL64), (np.float32, TOL32)):
        for fr in (None, (0.1, 0.3)):
            got = dsp.mt_cross_power_spectra(x.astype(dt), fs=1, demean=True, freq_range=fr, nw=3)
            want, f = op.mt_cross_power_spectra(x.astype(dt), fs=1.0, demean=True, freq_range=fr, nw=3)
            assert got.power.shape == want.shape and np.allclose(got.freq, f)
            assert relerr(got.power, want) < tol
            gc = dsp.mt_coherence(x.astype(dt), fs=1, demean=True, freq_range=fr, nw=3).coherence
            wc, _ = op.mt_coherence(x.astype(dt), fs=1.0, demean=True, freq_range=fr, nw=3)
            assert relerr(gc, wc) < 20 * tol


def test_hilbert_reference_cases():
    # test/util.jl:4-50
    from oracle.util import hilbert as hilbert_oracle
    t = np.arange(0, 2, 1 / 256)
    a0, a1, a2, a3 = np.sin(np.pi * t), np.cos(np.pi * t), np.sin(2 * np.pi * t), np.cos(2 * np.pi * t)
    a = np.stack([a0, a1, a2, a3], axis=1)
    h = np.stack([dsp.hilbert(a0), dsp.hilbert(a1), dsp.hilbert(a2), dsp.hilbert(a3)], axis=1)
    assert h.dtype == np.complex128
    assert relerr(h.real, a) < TOL64 and relerr(np.abs(h), np.ones(a.shape)) < TOL64
    assert np.allclose(np.angle(h[:256, 0]), -np.pi / 2 + np.pi / 256 * np.arange(256), atol=1e-9)
    assert np.allclose(np.angle(h[:256, 1]), np.pi / 256 * np.arange(256), atol=1e-9)
    assert np.allclose(np.angle(h[:128, 2]), -np.pi / 2 + np.pi / 128 * np.arange(128), atol=1e-9)
    assert np.allclose(np.angle(h[:128, 3]), np.pi / 128 * np.arange(128), atol=1e-9)
    assert relerr(h[:, 1].imag, a0) < TOL64                                  # Im hilbert(cos) = sin
    odd = np.concatenate([np.ones(10), np.zeros(9)])
    assert relerr(dsp.hilbert(odd).real, odd) < TOL64                        # odd length
    r = np.random.default_rng(3).integers(1, 21, 128)
    assert np.array_equal(dsp.hilbert(r), dsp.hilbert(r.astype(np.float64)))  # integers go through Float64
    assert relerr(dsp.hilbert(a), h) < TOL64                                 # 2-D: along dim 1
    with pytest.raises(dsp.ArgumentError):
        dsp.hilbert(a0 + 1j * a1)
    for n in (1, 2, 3, 8, 1000, 4099):
        for dt, tol in ((np.float32, TOL32), (np.float64, TOL64)):
            x = randn((n, 3), dt)
            y = dsp.hilbert(x)
            assert y.dtype == (np.complex64 if dt == np.float32 else np.complex128) and y.shape == x.shape
            assert relerr(y, hilbert_oracle(x.astype(np.float64))) < tol


def test_hilbert_device_resident():
    from oracle.util import hilbert as hilbert_oracle
    x = randn(1 << 16, np.float32)
    d = dsp.hilbert(dsp.to_device(x))
    assert isinstance(d, dsp.DeviceArray) and d.dtype == np.complex64
    assert relerr(dsp.to_host(d), hilbert_oracle(x.astype(np.float64))) < TOL32


@pytest.mark.parametrize("nb", [5, 31, 129])
def test_filtfilt_fir(nb):
    # src/Filters/filt.jl:301-325: zero-phase FIR filtering == extrapolate, filter with conv(b, reverse(b)), trim
    b = randn(nb, np.float64)
    for x in (randn(2000, np.float64), randn(4000, np.float64).reshape(2000, 2)):
        y = dsp.filtfilt(b, x)
        assert y.shape == x.shape
        x2 = x.reshape(2000, -1)
        newb = np.convolve(b, b[::-1])
        for c in range(x2.shape[1]):
            sig = x2[:, c]
            ext = np.concatenate([2 * sig[0] - sig[nb - 1:0:-1], sig, 2 * sig[-1] - sig[-2:-nb - 1:-1]])
            ref = od.filt(newb, 1.0, ext, f64=True)[2 * nb - 2:]
            assert relerr(y.reshape(2000, -1)[:, c], ref) < TOL64
    assert np.array_equal(dsp.filtfilt(b * 2.0, 2.0, x), dsp.filtfilt(b, x))


# =============================================================================== multitaper (SURVEY.md 8f rank 1)

def test_mt_pgram_matlab_goldens(goldens):
    # test/periodograms.jl:381-386, 404-486 (MATLAB pmtm)
    s = goldens["stft_x"]
    assert approx(dsp.mt_pgram(s, fs=16000).power, goldens["mt_pgram"])
    assert approx(dsp.mt_pgram(s, fs=16000, window=dsp.dpss(s.size, 4)).power, goldens["mt_pgram"])
    x = goldens["pmtm_x"]
    nfft = 1 << (x.size - 1).bit_length()
    r = dsp.mt_pgram(x, fs=1000, nw=4, nfft=nfft)
    assert approx(r.freq, goldens["pmtm_fx"]) and approx(r.power, goldens["pmtm_pxx"])
    assert relerr(r.power, op.mt_pgram(x, fs=1000, nw=4, nfft=nfft, f64=True)[0]) < TOL64
    cfg = dsp.MTConfig(np.float64, x.size, fs=1000, nw=4, nfft=nfft)
    assert np.array_equal(dsp.mt_pgram(x, cfg).power, r.power)
    r32 = dsp.mt_pgram(x.astype(np.float32), fs=1000, nw=4, nfft=nfft)
    assert r32.power.dtype == np.float32 and approx(r32.power, goldens["pmtm_pxx"])
    z = x + 1j * goldens["pmtm_y"]
    rz = dsp.mt_pgram(z, fs=1000, nw=4, nfft=nfft)
    m = (rz.freq > 0) & (rz.freq < 500)
    assert approx(rz.freq[m], goldens["pmtm_fz"][1:m.sum() + 1]) and approx(rz.power[m], goldens["pmtm_pzz"][1:m.sum() + 1])
    with pytest.raises(dsp.DimensionMismatch):
        dsp.mt_pgram(np.concatenate([x, [1.0]]), cfg)
    assert approx(dsp.dpss(128, 4), goldens["dpss128_4"])                      # test/windows.jl:32-36


def test_mt_spectrogram(goldens):
    # test/periodograms.jl:39-42: freq/time equal the plain spectrogram's, first column equals mt_pgram of the first segment
    x0 = goldens["spectrogram_x"]
    mt = dsp.mt_spectrogram(x0, 256, 128, fs=10)
    sp = dsp.spectrogram(x0, 256, 128, fs=10)
    assert np.array_equal(mt.freq, sp.freq) and np.array_equal(mt.time, sp.time)
    assert approx(mt.power[:, 0], dsp.mt_pgram(x0[:256], fs=10).power)
    ref, _, _ = op.mt_spectrogram(x0, 256, 128, fs=10, f64=True)
    assert relerr(mt.power, ref) < TOL64
    x = randn(40000, np.float32)
    mt32 = dsp.mt_spectrogram(x, 1000, 500, nw=3)                              # nfft = 1024 (fused), n = 1000
    ref32, _, _ = op.mt_spectrogram(x, 1000, 500, nw=3, f64=True)
    assert mt32.power.dtype == np.float32 and relerr(mt32.power, ref32) < TOL32


def test_unaligned_device_views_take_the_direct_load_path():
    # TMA bulk staging needs 16-byte aligned segment starts; a view that starts 8 bytes off must fall back to direct
    # loads and give the same spectrum as the aligned copy (complex64: one sample = 8 bytes; float32: 4 bytes)
    z = randn(200001, np.complex64)
    zd = dsp.to_device(z)
    cfg = dsp.WelchConfig(200000, np.complex64, n=1024, noverlap=512, window=dsp.hanning)
    a = dsp.welch_pgram(zd[1:], cfg).power
    assert np.array_equal(a, dsp.welch_pgram(z[1:], cfg).power)
    x = randn(150003, np.float32)
    xd = dsp.to_device(x)
    for off in (1, 2, 3):
        sp = dsp.spectrogram(xd[off:off + 150000], 512, 384).power.to_host()
        assert np.array_equal(sp, dsp.spectrogram(x[off:off + 150000], 512, 384).power)
        y = dsp.fftfilt(randn(300, np.float32) * 0 + 1, xd[off:off + 150000]).to_host()
        assert relerr(y, od.filt(np.ones(300, np.float32), np.float32(1), x[off:off + 150000], f64=True)) < TOL32


def test_edge_cases_empty_short_and_single_sample():
    # empty / too-short inputs follow the reference's conventions (no kernel launch, zero or empty results)
    assert dsp.filt([1.0, 2.0], 1.0, np.zeros(0)).shape == (0,)                              # src/dspbase.jl:39
    assert dsp.fftfilt(np.ones(70), np.zeros(0)).shape == (0,)
    p = dsp.welch_pgram(np.arange(5.0), 8, 4, window=None)                                   # k = 0 -> fill!(out, 0), :747
    assert p.power.shape == (5,) and not p.power.any()
    assert dsp.stft(np.arange(5.0), 8, 4).shape == (5, 0)
    sp = dsp.spectrogram(np.arange(5.0), 8, 4)
    assert sp.power.shape == (5, 0) and sp.time.size == 0
    assert dsp.arraysplit(np.arange(5.0), 8, 4).shape == (0, 8)
    # single-sample / single-segment / single-tap cases
    assert np.array_equal(dsp.conv(np.array([3.0]), np.array([2.0])), [6.0])
    assert np.array_equal(dsp.filt([2.0], 1.0, np.array([1.0, 2.0, 3.0])), [2.0, 4.0, 6.0])
    x = randn(4096, np.float32)
    one = dsp.welch_pgram(x, 4096, 2048, window=dsp.hanning)                                 # exactly one segment
    assert relerr(one.power, op.welch_pgram(x, 4096, 2048, window=ow.hanning, f64=True)[0]) < TOL32
    assert relerr(dsp.periodogram(x).power, op.periodogram(x, f64=True)[0]) < TOL32
    y = dsp.resample(np.array([1.0]), Fraction(3, 2))
    assert y.shape == (2,) and relerr(y, of.resample(np.array([1.0]), Fraction(3, 2))) < TOL64
    # filter longer than the signal (test/filt.jl uses xlen 127 with blen 127; here nb > nx)
    b = randn(300, np.float64)
    xs = randn(50, np.float64)
    assert relerr(dsp.fftfilt(b, xs), od.filt(b, 1.0, xs, f64=True)) < TOL64
    assert relerr(dsp.filt(b, 1.0, xs), od.filt(b, 1.0, xs, f64=True)) < TOL64
    assert relerr(dsp.conv(xs, b, algorithm="fft_overlapsave"), od.conv_exact(xs, b)) < TOL64
    # many channels at once (grid over columns)
    xm = randn(600 * 300, np.float32).reshape(600, 300)
    ym = dsp.fftfilt(randn(100, np.float32) * 0 + 0.01, xm)
    assert ym.shape == xm.shape and relerr(ym[:, 299], od.filt(np.full(100, 0.01, np.float32), np.float32(1), xm[:, 299], f64=True)) < TOL32
    rm = dsp.resample(xm, Fraction(2, 3), dims=0)
    assert rm.shape == (400, 300) and np.array_equal(rm[:, 17], dsp.resample(xm[:, 17], Fraction(2, 3)))


# =============================================================================== BASELINE configs 4 / 5 at their stated size

def test_spectrogram_config4_full_size_probes():
    # BASELINE configs[3] at its stated size: spectrogram of 64 channels x 2^22 Float32, n = nfft = 1024, noverlap = 768.
    # The output is 513 x 16381 x 64 Float32 = 2.15 GB (> 2^31 bytes: where a 32-bit index would wrap).  Checked by
    # (i) ~200 probe columns (corners of the (column, channel) grid + random) against the oracle run on that segment alone,
    # (ii) Parseval column by column for four whole channels (src/periodograms.jl:828-837, 872-897).
    rng = np.random.default_rng(4004)
    nchan, length, n, nov = 64, 1 << 22, 1024, 768
    hop = n - nov
    x = np.empty((length, nchan), dtype=np.float32, order="F")
    t = np.arange(length, dtype=np.float32) / np.float32(length)
    for c in range(nchan):
        x[:, c] = rng.standard_normal(length, dtype=np.float32) * np.float32(0.25)
        x[:, c] += np.cos(np.float32(2 * np.pi * (40000.0 + 9000.0 * c)) * t * (np.float32(1.0) + t))     # chirp per channel
    sp = dsp.spectrogram(x, n, nov)
    k = (length - n) // hop + 1
    assert sp.power.shape == (n // 2 + 1, k, nchan) and sp.power.dtype == np.float32 and k == 16381
    probes = [(0, 0), (k - 1, 0), (0, nchan - 1), (k - 1, nchan - 1), (k - 2, nchan - 1), (k // 2, nchan // 2)]
    probes += [(int(rng.integers(0, k)), int(rng.integers(0, nchan))) for _ in range(200)]
    worst = 0.0
    for col, c in probes:
        seg = x[col * hop: col * hop + n, c]
        truth, _, _ = op.spectrogram(seg, n, nov, f64=True)
        worst = max(worst, relerr(sp.power[:, col, c], truth[:, 0]))
    assert worst < TOL32, worst
    # Parseval: sum_k P[k, col] == sum_j x_j^2 over the segment (rectangular window, one-sided, fs = 1)
    for c in (0, 1, nchan // 2, nchan - 1):
        e = np.concatenate([[0.0], np.cumsum(x[:, c].astype(np.float64) ** 2)])
        seg_e = e[np.arange(k) * hop + n] - e[np.arange(k) * hop]
        tot = sp.power[:, :, c].sum(axis=0, dtype=np.float64)
        assert np.max(np.abs(tot - seg_e) / seg_e) < 2e-6
    assert sp.time[-1] == (n / 2 + hop * (k - 1))


def test_resample_config5_full_size_probes():
    # BASELINE configs[4] at its stated size: resample(x, 3//2) on 2^26 ComplexF32 (1.5 * 2^26 outputs), Float32 taps
    # (ComplexF32 out) and the default Float64 taps (ComplexF64 out, Appendix B).  An output depends on 37 input samples
    # only, so windows of the full-size result -- both ends and random interior ones -- are compared with the oracle run on
    # the matching input slice: y_full[j] = y_slice[j - 3 s0 / 2] for a slice starting at an even sample s0
    # (src/Filters/stream_filt.jl:476-515, 688-725).  The shift identity itself is first checked on the oracle alone.
    r = Fraction(3, 2)
    h64 = dsp.resample_filter(r)
    tpp = -(-h64.size // 3)
    xs = randn(6000, np.complex64)
    full = of.resample(xs, r, h64)
    part = of.resample(xs[2000:], r, h64)
    assert relerr(full[3000 + 2 * tpp:], part[2 * tpp:]) < 1e-14
    n = 1 << 26
    rng = np.random.default_rng(5005)
    x = np.empty(n, dtype=np.complex64)
    x.real = rng.standard_normal(n, dtype=np.float32)
    x.imag = rng.standard_normal(n, dtype=np.float32)
    win = 6000
    starts = [0, n - win] + [2 * int(rng.integers(1, (n - win) // 2)) for _ in range(6)]
    for h, out_dt, tolv in ((h64.astype(np.float32), np.complex64, TOL32), (h64, np.complex128, TOL64)):
        y = dsp.resample(x, r, h)
        assert y.dtype == out_dt and y.size == 3 * (n // 2)
        for s0 in starts:
            xs = x[s0:s0 + win] if s0 + win < n else x[s0:]
            ref = of.resample(xs, r, h, f64=True)
            j0 = 3 * s0 // 2
            lo = 0 if s0 == 0 else 2 * tpp                      # the slice's own start transient
            hi = ref.size if s0 + win >= n else ref.size - 2 * tpp   # ... and end transient (the last window runs to the end)
            assert relerr(y[j0 + lo:j0 + hi], ref[lo:hi]) < tolv, (out_dt, s0)
        del y


# =============================================================================== range (shard) forms of the C ABI

def test_os_exec_range_dev_reassembles_bit_equal():
    # dspb200_os_exec_range_dev: the stream cut into 8 contiguous OUTPUT ranges (each holding only its own input range +
    # the nv-1 halo, addressed by global offsets), run on one GPU and reassembled: bit-equal to the unsharded call when the
    # ranges are cut at multiples of the block length L (same blocks, same roundings), equal to rounding error otherwise
    from dspb200 import _lib, sharding
    for dt, nu, nv in ((np.complex64, 300001, 4097), (np.float32, 200000, 257), (np.complex128, 70001, 1025)):
        u, v = randn(nu, dt), randn(nv, dt)
        nout = nu + nv - 1
        plan = _lib.OsPlan(v, 0)
        du = dsp.to_device(u)
        whole = dsp.device.DeviceArray((nout,), dt)
        plan.exec_dev(du.ptr, nu, 1, whole.ptr, nout, 0)
        dsp.device.sync()
        ref = whole.to_host()
        truth = od.conv(u, v, f64=True)
        assert relerr(ref, truth) < tol(dt)
        for align in (plan.nfft - nv + 1, 1):
            got = np.full_like(ref, np.nan)
            for rank in range(8):
                sh = sharding.conv_shard(nu, nv, nout, 8, rank, align=align)
                local = dsp.to_device(u[sh.in_begin:sh.in_end])      # the rank holds nothing else
                part = dsp.device.DeviceArray((sh.out_count,), dt)
                plan.exec_range_dev(local.ptr, sh.in_begin, sh.in_end - sh.in_begin, part.ptr, sh.out_begin, sh.out_count, 0)
                dsp.device.sync()
                got[sh.out_begin:sh.out_begin + sh.out_count] = part.to_host()
            if align > 1:
                assert np.array_equal(got, ref), dt
            else:
                assert relerr(got, truth) < tol(dt), dt
        plan.close()


def test_resample_exec_range_dev_reassembles_bit_equal():
    # dspb200_resample_exec_range_dev: 8 output ranges, each given only the input samples it reads (global offsets)
    from dspb200 import _lib, sharding
    from dspb200.filters import resample_phase
    for tx, th, rate in ((np.complex64, np.float32, Fraction(3, 2)), (np.float32, np.float64, Fraction(5, 7)),
                         (np.complex128, np.float64, Fraction(2, 1))):
        x = randn(250001, tx)
        h = dsp.resample_filter(rate).astype(th)
        ref = dsp.resample(x, rate, h)
        n0, phi0 = resample_phase(h.size, rate)
        interp, decim = rate.numerator, rate.denominator
        tpp = -(-h.size // interp)
        plan = _lib.ResamplePlan(tx, h, interp, decim)
        got = np.empty_like(ref)
        for rank in range(8):
            sh = sharding.resample_shard(x.size, ref.size, interp, decim, n0, phi0, tpp, 8, rank)
            local = dsp.to_device(x[sh.in_begin:sh.in_end])
            part = dsp.device.DeviceArray((sh.out_count,), ref.dtype)
            plan.exec_range_dev(local.ptr, sh.in_begin, sh.in_end - sh.in_begin, n0, phi0, part.ptr, sh.j_begin, sh.out_count, 0)
            dsp.device.sync()
            got[sh.j_begin:sh.j_begin + sh.out_count] = part.to_host()
        assert np.array_equal(got, ref), (tx, th, rate)
        assert relerr(ref, of.resample(x, rate, h, f64=True)) < tol(ref.dtype)
        plan.close()


def test_welch_exec_range_dev_partials_sum_to_the_whole():
    # dspb200_welch_exec_range_dev: every "rank" transforms the segments that start in its sample range, scaled by the
    # GLOBAL 1/(k r); the sum of the 8 partial spectra (what the all-reduce forms) equals the unsharded PSD
    from dspb200 import _lib, sharding
    from dspb200.periodograms import compute_window
    for dt, length, n, nov, onesided in ((np.float32, 1 << 20, 4096, 2048, True), (np.complex64, 777777, 1024, 768, False),
                                         (np.float64, 300000, 2048, 1024, True)):
        s = randn(length, dt)
        whole = dsp.welch_pgram(s, n, nov, window=dsp.hanning, onesided=onesided)
        win, norm2 = compute_window(dsp.hanning, n)
        plan = _lib.SpecPlan(dt, n, nov, n, onesided, win)
        acc = np.zeros(whole.power.shape, dtype=np.float64)
        for rank in range(8):
            sh = sharding.welch_stream_shard(length, n, nov, 8, rank)
            if sh.seg_end <= sh.seg_begin:
                continue
            local = dsp.to_device(s[sh.sample_begin:sh.sample_end])
            part = dsp.device.DeviceArray(whole.power.shape, whole.power.dtype)
            plan.welch_range_dev(local.ptr, sh.sample_end - sh.sample_begin, sh.sample_begin, sh.seg_begin, sh.seg_end,
                                 sh.k_total * norm2, part.ptr, 0)
            dsp.device.sync()
            acc += part.to_host().astype(np.float64)
        assert relerr(acc, whole.power) < tol(dt), dt
        truth, _ = op.welch_pgram(s, n, nov, window=ow.hanning, onesided=onesided, f64=True)
        assert relerr(acc, truth) < tol(dt), dt
        plan.close()


def test_conv_integer_inputs_round_not_truncate():
    # conv of integer arrays through the FFT algorithms: the Float64 result is rounded (src/dspbase.jl:775-776), never
    # truncated toward zero (5.9999999 -> 6)
    rng = np.random.default_rng(77)
    u = rng.integers(-50, 50, 3000)
    v = rng.integers(-50, 50, 700)
    exact = np.convolve(u, v)
    for alg in ("direct", "fft", "fft_simple", "fft_overlapsave"):
        out = np.zeros(exact.size + 3, dtype=np.int64)
        dsp.conv_(out, u, v, algorithm=alg)
        assert np.array_equal(out[:exact.size], exact) and not out[exact.size:].any(), alg


def test_filtfilt_signal_as_long_as_the_filter():
    # filtfilt with length(x) == length(b): pad_length == n - 1 (src/Filters/filt.jl:245-259, 301-337)
    b = randn(9, np.float64)
    x = randn(9, np.float64)
    y = dsp.filtfilt(b, x)
    assert y.shape == x.shape
    ext = np.concatenate([2 * x[0] - x[8:0:-1], x, 2 * x[8] - x[7::-1][:8]])
    ref = np.convolve(ext, np.convolve(b, b[::-1]))[2 * 8: 2 * 8 + 9]
    assert relerr(y, ref) < 1e-12


def test_filt_welch_pipeline_matches_the_two_calls():
    # dspb200_filt_welch_exec: welch_pgram(filt(b, x), config) as one chunked host-pointer call -- same PSD as filtering and
    # estimating in two calls, and as the Float64 oracle (src/dspbase.jl:14-15, src/periodograms.jl:702-759); the streaming
    # entry points (begin / accumulate / finalize) are what it is made of
    from dspb200 import _lib
    for dt, n, nb in ((np.complex64, (1 << 23) + 12345, 1025), (np.float32, 3_000_001, 257), (np.float64, 400_000, 129)):
        x, b = randn(n, dt), randn(nb, dt)
        onesided = np.dtype(dt).kind != "c"
        cfg = dsp.WelchConfig(n, dt, n=4096, noverlap=2048, onesided=onesided, nfft=4096, window=dsp.hanning)
        p1 = dsp.filt_welch(x, b, cfg)
        y = dsp.conv(x, b, algorithm="fft_overlapsave")[:n]
        p2 = dsp.welch_pgram(y, cfg)
        assert p1.power.dtype == p2.power.dtype and relerr(p1.power, p2.power) < tol(dt)
        ytrue = od.conv(x.astype(np.complex128 if not onesided else np.float64), b.astype(np.complex128 if not onesided else np.float64),
                        f64=True)[:n]
        truth, _ = op.welch_pgram(ytrue, 4096, 2048, window=ow.hanning, onesided=onesided, f64=True)
        assert relerr(p1.power, truth) < tol(dt), dt
    # streaming Welch: three arbitrary segment chunks == one call
    s = randn(500_000, np.float32)
    cfg = dsp.WelchConfig(s.size, np.float32, n=1024, noverlap=512, window=dsp.hamming)
    whole = dsp.welch_pgram(s, cfg)
    k = (s.size - 1024) // 512 + 1
    d = dsp.to_device(s)
    out = dsp.device.DeviceArray(whole.power.shape, np.float32)
    cfg.plan.welch_begin_dev(0)
    for a, bnd in ((0, 100), (100, 101), (101, k)):
        cfg.plan.welch_accumulate_dev(d.ptr, s.size, 0, a, bnd, 0)
    cfg.plan.welch_finalize_dev(k * cfg.r, out.ptr, 0)
    dsp.device.sync()
    assert relerr(out.to_host(), whole.power) < TOL32
