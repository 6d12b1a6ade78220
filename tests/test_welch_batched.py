"""Batched welch_pgram: a len x nchan matrix whose columns are independent channels, Welch-averaged in one call
(dspb200_welch_batch_exec / _dev).  The reference's welch_pgram takes a vector only, so every column is checked against the
double-precision oracle run on that column alone -- per column, never over the whole matrix, so that a large channel cannot
hide a broken small one."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT, relerr

import dspb200 as dsp
from oracle import periodograms as op
from oracle import windows as ow

TOL32 = 1e-6
TOL64 = 1e-12


def tol(dt):
    return TOL32 if np.dtype(dt) in (np.dtype(np.float32), np.dtype(np.complex64)) else TOL64


def randn(rng, shape, dt):
    dt = np.dtype(dt)
    if dt.kind == "c":
        return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(dt)
    return rng.standard_normal(shape).astype(dt)


def check_columns(P, S, dt, **kw):
    """Every column of P within tol(dt) of the Float64 oracle on the same column of S."""
    assert P.dtype == dsp.fftabs2type(dt) and P.shape[1] == S.shape[1]
    for c in range(S.shape[1]):
        truth, _ = op.welch_pgram(S[:, c], f64=True, **kw)
        assert P.shape[0] == truth.shape[0]
        if not truth.any():
            assert not P[:, c].any(), f"column {c}: expected zeros"
            continue
        e = relerr(P[:, c], truth)
        assert e < tol(dt), f"column {c}: relerr {e:.3e}"


# =============================================================================== CPU: interface and argument checks

def test_batch_symbols_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "dspb200.h")).read()
    for name in ("dspb200_welch_batch_exec", "dspb200_welch_batch_exec_dev"):
        assert re.search(r"DSPB200_API\s+int\s+" + name + r"\s*\(", hdr), name
        assert name in dsp._lib.SIGNATURES
        assert hasattr(dsp._lib.lib, name)


class _StubPlan:
    """Stands in for the device plan: the checks under test must fail before any library call."""

    def __init__(self, dtype, n, noverlap, nfft, onesided, window=None):
        self.nout = nfft // 2 + 1 if onesided else nfft

    def __getattr__(self, name):
        raise AssertionError(f"the library was reached ({name})")


def test_matrix_argument_checks_before_the_library(monkeypatch):
    from dspb200 import periodograms as pg
    monkeypatch.setattr(pg._lib, "SpecPlan", _StubPlan)
    S = np.zeros((256, 3), dtype=np.float32)
    cfg = dsp.WelchConfig(S, n=64, noverlap=32, window=None)
    assert cfg.nsamples == 64 and cfg.freq.size == 33
    # WelchConfig(S) takes nsamples from the rows: default n = size(s, 1) >> 3
    assert dsp.WelchConfig(S, window=None).nsamples == 256 >> 3
    with pytest.raises(dsp.DimensionMismatch):
        dsp.welch_pgram_(np.zeros((33, 2), np.float32), S, cfg)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.welch_pgram_(np.zeros((32, 3), np.float32), S, cfg)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.welch_pgram_(np.zeros(33 * 3, np.float32), S, cfg)
    with pytest.raises(dsp.ArgumentError):
        dsp.welch_pgram_(np.zeros((33, 3), np.float64), S, cfg)
    with pytest.raises(dsp.ArgumentError):
        dsp.welch_pgram_(np.zeros((33, 3), np.float64), S.astype(np.float64), cfg)
    with pytest.raises(dsp.ArgumentError):
        dsp.welch_pgram(S.astype(np.complex64), 64, 32, onesided=True, window=None)
    with pytest.raises(dsp.DomainError):
        dsp.welch_pgram(S, 64, 64, window=None)
    with pytest.raises(dsp.DomainError):
        dsp.welch_pgram(S, 64, 32, nfft=32, window=None)
    with pytest.raises(dsp.DomainError):
        dsp.welch_pgram_(np.zeros((33, 3), np.float32), S, 64, -1)
    # k == 0 and nchan == 0 return zeros without a launch
    p = dsp.welch_pgram(S[:10], cfg)
    assert p.power.shape == (33, 3) and not p.power.any()
    p = dsp.welch_pgram(np.zeros((256, 0), np.float32), cfg)
    assert p.power.shape == (33, 0)


# =============================================================================== GPU

SIZES = [(256, 128, 256), (1024, 512, 1024), (4096, 2048, 4096), (16384, 8192, 16384), (400, 240, 500)]
# (segments per channel, window, onesided): odd and even counts, one segment, none
VARIANTS = [(37, None, None), (38, "hanning", False), (1, "hanning", None), (0, None, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64, np.complex64, np.complex128])
@pytest.mark.parametrize("n,nov,nfft", SIZES)
@pytest.mark.parametrize("nchan", [1, 3, 64])
def test_batched_columns_vs_oracle(dt, n, nov, nfft, nchan):
    if np.dtype(dt).itemsize == 8 * (2 if np.dtype(dt).kind == "c" else 1) and nfft == 16384:
        n, nov, nfft = 8192, 4096, 8192
    rng = np.random.default_rng(n + nchan)
    hop = n - nov
    cplx = np.dtype(dt).kind == "c"
    for k, win, onesided in VARIANTS:
        if cplx:
            onesided = False
        length = n + hop * (k - 1) + 5 if k > 0 else n - 1
        S = randn(rng, (length, nchan), dt) * (1.0 + np.arange(nchan))
        S = S.astype(dt)
        p = dsp.welch_pgram(S, n, nov, onesided=onesided, nfft=nfft, fs=2.5,
                            window={None: None, "hanning": dsp.hanning}[win])
        nout = nfft // 2 + 1 if (onesided if onesided is not None else not cplx) else nfft
        assert p.power.shape == (nout, nchan)
        assert p.freq.size == nout
        check_columns(p.power, S, dt, n=n, noverlap=nov, onesided=onesided, nfft=nfft, fs=2.5,
                      window={None: None, "hanning": ow.hanning}[win])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.complex64, np.float64])
def test_channels_do_not_leak(dt):
    # one tone per channel at its own bin, channels scaled by powers of ten: segments of two channels sharing an FFT, a wrong
    # channel stride or a partial row added to the wrong channel moves a peak or breaks a column's oracle check
    nchan, n, nov = 8, 1024, 512
    length = n + (n - nov) * 40 + 7                                  # 41 segments: odd, the last real unit half filled
    t = np.arange(length)
    rng = np.random.default_rng(5)
    S = np.empty((length, nchan), dtype=dt)
    bins = [37 + 53 * c for c in range(nchan)]
    for c in range(nchan):
        ph = 2 * np.pi * bins[c] / n * t
        x = (np.exp(1j * ph) if np.dtype(dt).kind == "c" else np.cos(ph)) + 0.01 * rng.standard_normal(length)
        S[:, c] = (x * 10.0 ** (c - 3)).astype(dt)
    p = dsp.welch_pgram(S, n, nov, window=dsp.hanning)
    for c in range(nchan):
        assert int(np.argmax(p.power[:, c])) == bins[c], c
    check_columns(p.power, S, dt, n=n, noverlap=nov, window=ow.hanning)


@pytest.mark.gpu
def test_many_short_channels_one_slice_each():
    # more channels than resident virtual CTAs: one slice per channel, several items per virtual CTA
    rng = np.random.default_rng(11)
    n = 1024
    S = rng.standard_normal((2 * n, 1000)).astype(np.float32)
    p = dsp.welch_pgram(S, n, n // 2, window=dsp.hanning)
    check_columns(p.power, S, np.float32, n=n, noverlap=n // 2, window=ow.hanning)


@pytest.mark.gpu
def test_long_channels_split_into_slices():
    rng = np.random.default_rng(12)
    S = rng.standard_normal((1 << 22, 2)).astype(np.float32)
    p = dsp.welch_pgram(S, 4096, 2048, window=dsp.hanning)
    check_columns(p.power, S, np.float32, n=4096, noverlap=2048, window=ow.hanning)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_channel_groups_past_the_scratch_bound(dt):
    # 64 KB rows (16384-point Float32, 8192-point Float64): the 32 MiB scratch holds 512 of them, so 600 channels run in two
    # channel groups
    rng = np.random.default_rng(13)
    n = 16384 if dt == np.float32 else 8192
    S = rng.standard_normal((2 * n, 600)).astype(dt)
    p = dsp.welch_pgram(S, n, n // 2, window=None)
    check_columns(p.power, S, dt, n=n, noverlap=n // 2, window=None)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.complex64])
def test_unaligned_channel_stride_matches_aligned(dt):
    # an odd len puts every channel after the first off 16-byte alignment: the direct-load (non-TMA) instance
    rng = np.random.default_rng(14)
    n, nov = 4096, 2048
    A = randn(rng, (n + 2048 * 20 + 3, 5), dt)                     # odd len
    B = np.asfortranarray(np.vstack([A, np.zeros((1, 5), dt)]))     # even len, same segments
    pa = dsp.welch_pgram(A, n, nov, window=dsp.hanning, onesided=False)
    pb = dsp.welch_pgram(B, n, nov, window=dsp.hanning, onesided=False)
    for c in range(5):
        assert relerr(pa.power[:, c], pb.power[:, c]) < tol(dt)
    check_columns(pa.power, A, dt, n=n, noverlap=nov, window=ow.hanning, onesided=False)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.complex128])
def test_device_input_and_repeat_calls_bit_equal(dt):
    rng = np.random.default_rng(15)
    S = np.asfortranarray(randn(rng, (1 << 16, 6), dt))
    cfg = dsp.WelchConfig(S, n=1024, noverlap=512, window=dsp.hanning)
    a = dsp.welch_pgram(S, cfg).power
    b = dsp.welch_pgram(S, cfg).power
    assert np.array_equal(a, b)
    d = dsp.welch_pgram(dsp.to_device(S), cfg).power
    assert np.array_equal(a, d)
    out = np.empty_like(a)
    assert np.array_equal(dsp.welch_pgram_(out, S, cfg).power, a)
    check_columns(a, S, dt, n=1024, noverlap=512, window=ow.hanning)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64, np.complex64, np.complex128])
def test_one_channel_matches_the_vector_form(dt):
    rng = np.random.default_rng(16)
    x = randn(rng, 300001, dt)
    v = dsp.welch_pgram(x, 4096, 2048, window=dsp.hanning, onesided=False).power
    m = dsp.welch_pgram(x[:, None], 4096, 2048, window=dsp.hanning, onesided=False).power
    assert m.shape == (4096, 1)
    assert relerr(m[:, 0], v) < tol(dt)
    print(f"{np.dtype(dt)}: batched nchan=1 bit-equal to the vector form: {np.array_equal(m[:, 0], v)}")


@pytest.mark.gpu
def test_streaming_accumulation_survives_a_batch():
    # welch_begin / accumulate ... batch ... accumulate / finalize: the batch has its own scratch
    rng = np.random.default_rng(17)
    s = rng.standard_normal(1 << 18).astype(np.float32)
    S = rng.standard_normal((1 << 16, 4)).astype(np.float32)
    cfg = dsp.WelchConfig(s, n=4096, noverlap=2048, window=dsp.hanning)
    whole = dsp.welch_pgram(s, cfg).power
    k = dsp.arraysplit_count(s.size, 4096, 2048)
    d = dsp.to_device(s)
    out = dsp.DeviceArray(whole.shape, whole.dtype)
    cfg.plan.welch_begin_dev(0)
    cfg.plan.welch_accumulate_dev(d.ptr, s.size, 0, 0, k // 2, 0)
    batch = dsp.welch_pgram(S, cfg).power
    cfg.plan.welch_accumulate_dev(d.ptr, s.size, 0, k // 2, k, 0)
    cfg.plan.welch_finalize_dev(k * cfg.r, out.ptr, 0)
    assert relerr(out.to_host(), whole) < TOL32
    check_columns(batch, S, np.float32, n=4096, noverlap=2048, window=ow.hanning)


@pytest.mark.gpu
def test_config3_across_channels_and_reference_budget():
    # BASELINE config 3 (4096 / 50 % / hanning, Float32) on 8 channels of 2^22: every column within 1e-6 of the Float64 truth
    # and no worse than the reference's own sequential Float32 loop (test_welch_config3_scaled_and_reference_budget's budget)
    rng = np.random.default_rng(1003)
    n, nchan = 1 << 22, 8
    t = np.arange(n)
    S = np.empty((n, nchan), dtype=np.float32, order="F")
    for c in range(nchan):
        S[:, c] = (rng.standard_normal(n) + np.cos(2 * np.pi * (0.1 + 0.01 * c) * t)
                   + 0.1 * np.cos(2 * np.pi * 0.2345 * t)).astype(np.float32)
    p = dsp.welch_pgram(S, 4096, 2048, window=dsp.hanning)
    assert p.power.shape == (2049, nchan) and p.power.dtype == np.float32
    for c in range(nchan):
        truth, _ = op.welch_pgram(S[:, c], 4096, 2048, window=ow.hanning, f64=True)
        ref32, _ = op.welch_pgram(S[:, c], 4096, 2048, window=ow.hanning, sequential=True)
        e_gpu, e_ref = relerr(p.power[:, c], truth), relerr(ref32, truth)
        assert e_gpu < TOL32 and e_gpu <= 1.5 * e_ref + 1e-7, (c, e_gpu, e_ref)
