"""Multitaper periodograms and spectrograms of channel matrices: mt_pgram / mt_spectrogram of a len x nchan matrix
(dspb200_mt_pgram_batch_exec(_dev), dspb200_mt_spectrogram_batch_exec(_dev)), whose columns are independent channels.

Every channel's tapers are summed in taper order, so at fused sizes column c of a matrix call has the bits of
  * mt_spectrogram: the Float32 / Float64 sum in taper order of the batched `spectrogram` of the same matrix under each taper
    row (window w_t / sqrt(r_t), r = 1), and of the vector call on that column -- except Float32 nfft = 1024 when the
    matrix's channels are off 16-byte alignment: the matrix call then runs stft_fused_kernel and the vector call the
    warp-per-unit kernel, which round differently (as for the batched spectrogram);
  * mt_pgram: the vector call on that column, wherever the column sits in a matrix of any width, on every pinned instance.
cuFFT sizes are checked against the per-bin bound of DESIGN.md section 4 with m = ntapers."""
import math
import os
import re

import numpy as np
import pytest

from conftest import ROOT

import dspb200 as dsp
import test_spectral_kernel_paths as kp
from test_spectral_kernel_paths import F32, F64, C64, C128, Guarded, same_bits

TAPER_SETS = (1, 2, 7)


def mt_fused(dt, nfft):
    """The fused / cuFFT routing of a multitaper plan, as for every spectral plan (fused_size_ok, spectral.cu)."""
    return kp.fused_size_ok(nfft, kp._f64(dt))


def mt_launches(fused, kind, nchan, ntapers, nfft, k=1):
    """Launches of one call: fused mt_spectrogram 1, fused mt_pgram 2 per channel group (one group below 32 MiB of partial
    rows), cuFFT mt_pgram 3 per batch of (channel, taper) pairs plus the scaling, cuFFT mt_spectrogram 3 per batch of
    (channel, segment) pairs per taper plus one add per taper after the first."""
    if nchan == 0 or k == 0:
        return 0
    if fused:
        return 1 if kind == "spectrogram" else 2
    b = kp.generic_batch(nfft)
    if kind == "pgram":
        return 3 * kp.cdiv(nchan * ntapers, b) + 1
    return ntapers * 3 * kp.cdiv(nchan * k, b) + ntapers - 1


def tapers(n, nt):
    """nt unit-energy Slepian rows, so that r_t = 1 and the rows are their own pre-scaled form."""
    return kp._tapers(n, nt)


# =============================================================================== CPU

def test_batch_symbols_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "dspb200.h")).read()
    for name in ("dspb200_mt_pgram_batch_exec", "dspb200_mt_pgram_batch_exec_dev", "dspb200_mt_spectrogram_batch_exec",
                 "dspb200_mt_spectrogram_batch_exec_dev"):
        assert re.search(r"DSPB200_API\s+int\s+" + name + r"\s*\(", hdr), name
        assert name in dsp._lib.SIGNATURES
        assert hasattr(dsp._lib.lib, name)


class _StubMtPlan:
    """Stands in for the device plan: records the calls the front end makes (host arrays only: no device form)."""
    calls = []
    mt_pgram_batch_dev = mt_spectrogram_batch_dev = None

    def __init__(self, dtype, n, noverlap, nfft, onesided, tapers):
        self.nout = nfft // 2 + 1 if onesided else nfft
        self.ntapers = tapers.shape[0]

    def mt_pgram_batch(self, s, length, nchan, out):
        assert s.flags.f_contiguous and s.shape == (length, nchan) and out.shape[0] == self.nout
        _StubMtPlan.calls.append(("pgram", s.dtype, length, nchan, out.shape))
        out[...] = 1

    def mt_spectrogram_batch(self, s, length, nchan, out):
        assert s.flags.f_contiguous and s.shape == (length, nchan) and out.shape[0] == self.nout
        _StubMtPlan.calls.append(("spectrogram", s.dtype, length, nchan, out.shape))
        out[...] = 1

    def __getattr__(self, name):
        raise AssertionError(f"the library was reached ({name})")


def test_front_end_shapes_eltypes_and_refusals(monkeypatch):
    from dspb200 import multitaper as mtm
    monkeypatch.setattr(mtm._lib, "MtPlan", _StubMtPlan)
    calls = _StubMtPlan.calls
    calls.clear()
    S = np.ones((64, 3), dtype=np.float32)
    p = dsp.mt_pgram(S, nw=2)
    assert p.power.shape == (33, 3) and p.power.dtype == np.float32 and p.freq.size == 33
    assert calls[-1] == ("pgram", np.dtype(np.float32), 64, 3, (33, 3))
    p = dsp.mt_pgram(S[:, 0], nw=2)                                   # a vector keeps its shape
    assert p.power.shape == (33,) and calls[-1][3] == 1
    p = dsp.mt_pgram(S.astype(np.int16), nw=2)                        # integer samples run as Float64
    assert p.power.dtype == np.float64 and calls[-1][1] == np.dtype(np.float64)
    p = dsp.mt_pgram(S.astype(np.complex64), nw=2)
    assert p.power.shape == (64, 3) and p.power.dtype == np.float32
    cfg = dsp.MTConfig(np.float32, 64, nw=2)
    assert dsp.mt_pgram(S, cfg).power.shape == (33, 3)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.mt_pgram(np.ones((65, 3), np.float32), cfg)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_pgram(np.ones((64, 3, 2), np.float32), nw=2)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_spectrogram(np.ones((64, 3, 2), np.float32), 16, 8, nw=2)
    n_before = len(calls)
    p = dsp.mt_pgram(np.ones((64, 0), np.float32), cfg)              # no channel: zeros, no call
    assert p.power.shape == (33, 0) and len(calls) == n_before
    # spectrogram: nout x k x nchan, freq and time from len = size(S, 1)
    L = 200
    sp = dsp.mt_spectrogram(np.ones((L, 4), np.float64), 32, 24, nw=2, fs=2.0)
    k = (L - 32) // 8 + 1
    assert sp.power.shape == (17, k, 4) and sp.power.dtype == np.float64
    assert calls[-1] == ("spectrogram", np.dtype(np.float64), L, 4, (17, k, 4))
    assert np.allclose(sp.time, (16 + 8 * np.arange(k)) / 2.0) and sp.freq.size == 17
    sv = dsp.mt_spectrogram(np.ones(L, np.float64), 32, 24, nw=2)
    assert sv.power.shape == (17, k)
    n_before = len(calls)
    sp = dsp.mt_spectrogram(np.ones((20, 4), np.float32), 32, 24, nw=2)   # no segment
    assert sp.power.shape == (17, 0, 4) and len(calls) == n_before
    sp = dsp.mt_spectrogram(np.ones((L, 0), np.float32), 32, 24, nw=2)    # no channel
    assert sp.power.shape == (17, k, 0) and len(calls) == n_before
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_spectrogram(np.ones((L, 2), np.float32), 32, 32, nw=2)


def test_restated_routing_and_launch_counts():
    assert [n for n in (200, 256, 1000, 1024, 8192, 16384, 32768) if mt_fused(F32, n)] == [256, 1024, 8192, 16384]
    assert not mt_fused(F64, 16384) and mt_fused(C128, 8192)
    # the C4-shaped 64-channel, 7-taper spectrogram: one launch (per-taper launches: 64 x 7 = 448)
    assert mt_launches(True, "spectrogram", 64, 7, 1024, k=(1 << 22) // 256 - 3) == 1
    assert mt_launches(True, "pgram", 1024, 7, 2048) == 2
    assert mt_launches(False, "pgram", 64, 7, 65536) == 3 * kp.cdiv(64 * 7, 64) + 1
    assert mt_launches(False, "spectrogram", 3, 7, 1000, k=5) == 7 * 3 + 6
    assert mt_launches(True, "pgram", 0, 7, 2048) == 0 and mt_launches(True, "spectrogram", 3, 7, 1024, k=0) == 0


# =============================================================================== GPU helpers

def _mt_plan(dt, n, hop, nfft, nt):
    plan = dsp._lib.MtPlan(dt, n, n - hop, nfft, not kp._cplx(dt), tapers(n, nt))
    assert plan.fused == mt_fused(dt, nfft)
    return plan


def _launches(f):
    n0 = dsp.launch_count()
    r = f()
    from dspb200 import device
    device.sync()
    return r, dsp.launch_count() - n0


def _mt_spec_dev(plan, gin, length, nchan, k):
    go = Guarded(kp._real(plan.dtype), plan.nout * k * nchan)
    _, nl = _launches(lambda: plan.mt_spectrogram_batch_dev(gin.ptr, length, nchan, go.ptr, 0))
    gin.data()
    return go.data((plan.nout, k * nchan)), nl


def _mt_pgram_dev(plan, gin, nchan):
    go = Guarded(kp._real(plan.dtype), plan.nout * nchan)
    _, nl = _launches(lambda: plan.mt_pgram_batch_dev(gin.ptr, plan.n, nchan, go.ptr, 0))
    gin.data()
    return go.data((plan.nout, nchan)), nl


def _taper_sum(dt, n, hop, nfft, rows, gin, length, nchan, k):
    """The Float32 / Float64 sum in taper order of the batched spectrogram under each taper row (r = 1)."""
    acc = None
    for w in rows:
        p = kp._plan(dsp, dt, n, hop, nfft, not kp._cplx(dt), w)
        try:
            col = kp._stft(dsp, p, gin, length, nchan, 1.0, 1, p.nout, k)
        finally:
            p.close()
        acc = col if acc is None else (acc + col).astype(kp._real(dt))
    return acc


# (dt, nfft, n, hop, k, nt, nchan, odd): odd len puts the channels of a matrix off 16-byte alignment (direct loads)
SPEC_CASES = [
    (F32, 1024, 1024, 256, 9, 7, 3, False),       # stft_w1k_kernel, TMA
    (F32, 1024, 1024, 256, 8, 7, 3, True),        # stft_fused_kernel, direct loads
    (F32, 1024, 1000, 250, 7, 2, 70, False),      # n < nfft, 70 channels
    (C64, 1024, 1024, 512, 6, 2, 3, False),       # complex 1024-point, warp kernel
    (C64, 1024, 1024, 512, 5, 7, 3, True),
    (F32, 256, 256, 64, 11, 7, 70, False),
    (F32, 2048, 2048, 512, 6, 1, 1, False),
    (F32, 4096, 3000, 1000, 5, 2, 3, True),
    (F32, 8192, 8192, 2048, 4, 7, 3, False),
    (F32, 8192, 8192, 4096, 3, 2, 3, True),
    (F32, 16384, 16384, 4096, 3, 2, 3, False),
    (C64, 2048, 2048, 1024, 5, 7, 3, False),
    (C64, 16384, 16000, 8000, 2, 2, 1, False),
    (F64, 512, 512, 128, 9, 7, 70, True),
    (F64, 8192, 8192, 4096, 3, 2, 3, False),
    (C128, 256, 200, 100, 6, 7, 3, False),
    (C128, 4096, 4096, 1024, 4, 1, 3, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,nfft,n,hop,k,nt,nchan,odd", SPEC_CASES,
                         ids=[f"{c[0].name}-{c[1]}-n{c[2]}-k{c[4]}-t{c[5]}-c{c[6]}{'-odd' if c[7] else ''}" for c in SPEC_CASES])
def test_mt_spectrogram_fused_is_the_taper_sum(dt, nfft, n, hop, k, nt, nchan, odd):
    from dspb200 import device
    rng = np.random.default_rng([nfft, n, k, nt, nchan, dt.num])
    length = (k - 1) * hop + n + (1 if odd else 0)
    S = np.asfortranarray(kp.signal(rng, (length, nchan), dt))
    plan = _mt_plan(dt, n, hop, nfft, nt)
    rows = tapers(n, nt)
    try:
        gin = Guarded(dt, length * nchan, rng, S)
        got, nl = _mt_spec_dev(plan, gin, length, nchan, k)
        assert nl == mt_launches(True, "spectrogram", nchan, nt, nfft, k)
        assert not np.isnan(got).any()
        assert same_bits(got, _taper_sum(dt, n, hop, nfft, rows, gin, length, nchan, k))
        # the vector call on a column: the same bits unless the kernel family differs (module docstring)
        family_differs = dt in (F32, C64) and nfft == 1024 and odd and nchan > 1 and (length * dt.itemsize) % 16 != 0
        for c in ({0, nchan // 2, nchan - 1}):
            gv = Guarded(dt, length, rng, S[:, c])
            vec, nlv = _mt_spec_dev(plan, gv, length, 1, k)
            assert nlv == 1
            if not family_differs:
                assert same_bits(vec, got[:, c * k:(c + 1) * k]), c
        host = np.full((plan.nout, k, nchan), np.nan, dtype=kp._real(dt), order="F")
        plan.mt_spectrogram_batch(S, length, nchan, host)
        assert same_bits(host.reshape(plan.nout, k * nchan, order="F"), got)
    finally:
        plan.close()
        device.empty_cache()


# (dt, N, n, nchan): the fused mt_pgram sizes
PGRAM_CASES = [(F32, 256, 256, 70), (F32, 1024, 1024, 3), (F32, 2048, 2000, 70), (F32, 4096, 4096, 3), (F32, 8192, 8192, 3),
               (F32, 16384, 16384, 3), (C64, 1024, 1024, 70), (C64, 4096, 3001, 3), (F64, 512, 512, 3), (F64, 8192, 8192, 3),
               (C128, 2048, 2048, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N,n,nchan", PGRAM_CASES, ids=[f"{c[0].name}-{c[1]}-n{c[2]}-c{c[3]}" for c in PGRAM_CASES])
def test_mt_pgram_columns_are_the_vector_call(dt, N, n, nchan):
    from dspb200 import device
    rng = np.random.default_rng([N, n, nchan, dt.num, 2])
    onesided = not kp._cplx(dt)
    for nt in TAPER_SETS:
        rows = tapers(n, nt)
        S = np.asfortranarray(kp.signal(rng, (n, nchan), dt) * (1.0 + np.arange(nchan)).astype(kp._real(dt)))
        plan = _mt_plan(dt, n, n, N, nt)
        try:
            gin = Guarded(dt, n * nchan, rng, S)
            P, nl = _mt_pgram_dev(plan, gin, nchan)
            assert nl == mt_launches(True, "pgram", nchan, nt, N)
            vec = []
            for c in range(nchan) if nchan <= 3 else (0, 1, 37, nchan - 1):
                v, _ = _mt_pgram_dev(plan, Guarded(dt, n, rng, S[:, c]), 1)
                assert same_bits(v[:, 0], P[:, c]), (nt, c)
                vec.append((c, v[:, 0]))
                X = np.concatenate([kp.ref_segments(S[:, c], n, n, N, rows[t])[0] for t in range(nt)])
                en = np.concatenate([kp.ref_segments(S[:, c], n, n, N, rows[t])[1] for t in range(nt)])
                kp._note(dt, kp.check_welch(P[:, c], X, en, N, onesided, 1.0, kp.eps(dt), nt, ("mt_pgram", nt, c)))
            # a column moved to another position in a matrix of another width keeps its bits
            c, v = vec[-1]
            S2 = np.asfortranarray(np.concatenate([kp.signal(rng, (n, 2), dt), S[:, c:c + 1]], axis=1))
            P2, _ = _mt_pgram_dev(plan, Guarded(dt, n * 3, rng, S2), 3)
            assert same_bits(P2[:, 2], v)
            host = np.full((plan.nout, nchan), np.nan, dtype=kp._real(dt), order="F")
            plan.mt_pgram_batch(S, n, nchan, host)
            assert same_bits(host, P)
            # every batched instance that can address a taper row, pinned: the same bits, and it is the one that ran
            fit = [mg for mg in kp.welch_instances(dt, N) if mg[0] <= 1 and kp.welch_smem(dt, N, mg[0], n, n, mg[1]) <= kp.SMEM_OPTIN]
            aligned = (n * dt.itemsize) % 16 == 0
            for mode, g in fit:
                plan.pin_welch(1, mode, g, 6 * g)
                Pp, _ = _mt_pgram_dev(plan, gin, nchan)
                assert same_bits(Pp, P), (nt, mode, g)
                assert plan.welch_config(2, aligned)[:2] == ((mode, g) if aligned else (0, 1))
            plan.pin_welch(1, -1, 0, 0)
        finally:
            plan.close()
            device.empty_cache()


# (dt, nfft, n): cuFFT sizes, n < nfft
GENERIC = [(F32, 1000, 900), (C64, 2000, 1999), (F32, 24000, 20000), (F64, 2000, 1500)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,nfft,n", GENERIC, ids=[f"{c[0].name}-{c[1]}" for c in GENERIC])
def test_mt_cufft_sizes_within_the_bound(dt, nfft, n):
    from dspb200 import device
    rng = np.random.default_rng([nfft, n, dt.num, 3])
    onesided = not kp._cplx(dt)
    nt, nchan = 7, 5
    rows = tapers(n, nt)
    S = np.asfortranarray(kp.signal(rng, (n, nchan), dt))
    plan = _mt_plan(dt, n, n, nfft, nt)
    identical = True
    try:
        gin = Guarded(dt, n * nchan, rng, S)
        P, nl = _mt_pgram_dev(plan, gin, nchan)
        assert nl == mt_launches(False, "pgram", nchan, nt, nfft)
        for c in range(nchan):
            segs = [kp.ref_segments(S[:, c], n, n, nfft, rows[t]) for t in range(nt)]
            X, en = np.concatenate([s[0] for s in segs]), np.concatenate([s[1] for s in segs])
            kp._note(dt, kp.check_welch(P[:, c], X, en, nfft, onesided, 1.0, kp.eps(dt), nt, ("cufft mt_pgram", c)))
            v, _ = _mt_pgram_dev(plan, Guarded(dt, n, rng, S[:, c]), 1)
            identical &= same_bits(v[:, 0], P[:, c])
    finally:
        plan.close()
    # spectrogram: hop n / 2, three segments per channel
    hop, k = n // 2, 3
    length = (k - 1) * hop + n
    S = np.asfortranarray(kp.signal(rng, (length, nchan), dt))
    plan = _mt_plan(dt, n, hop, nfft, nt)
    try:
        gin = Guarded(dt, length * nchan, rng, S)
        got, nl = _mt_spec_dev(plan, gin, length, nchan, k)
        assert nl == mt_launches(False, "spectrogram", nchan, nt, nfft, k)
        assert same_bits(got, _taper_sum(dt, n, hop, nfft, rows, gin, length, nchan, k))
        b, mult = kp.bins_and_mult(nfft, onesided)
        for c in range(nchan):
            for j in range(k):
                x = S[j * hop:j * hop + n, c]
                segs = [kp.ref_segments(x, n, n, nfft, rows[t]) for t in range(nt)]
                Sbin = sum(np.abs(s[0][0, b]) ** 2 for s in segs)
                E = float(sum(s[1][0] for s in segs))
                kp._note(dt, kp.check_power(got[:, c * k + j], Sbin, E, mult, 1.0, kp.eps(dt), nfft, nt, ("cufft mt_spec", c, j)))
            gv = Guarded(dt, length, rng, S[:, c])
            vec, _ = _mt_spec_dev(plan, gv, length, 1, k)
            identical &= same_bits(vec, got[:, c * k:(c + 1) * k])
    finally:
        plan.close()
        device.empty_cache()
    print(f"cuFFT {dt.name} nfft {nfft}: matrix columns bit-identical to the vector calls: {identical}")


@pytest.mark.gpu
def test_c_abi_refusals_launch_nothing():
    from dspb200 import device
    lib, check = dsp._lib.lib, dsp._lib.check
    n, nt, nchan = 1024, 3, 4
    plan = _mt_plan(F32, n, n, n, nt)
    spec = dsp._lib.MtPlan(F32, 256, 128, 256, True, tapers(256, nt))
    try:
        s = device.to_device(np.ones(n * nchan, np.float32))
        out = device.DeviceArray((plan.nout * nchan,), np.float32)
        n0 = dsp.launch_count()
        for args in ((None, n, nchan, out.ptr), (s.ptr, n, nchan, None), (s.ptr, n + 1, nchan, out.ptr), (s.ptr, n, -1, out.ptr),
                     (s.ptr, n, nchan, s.ptr + 64)):
            with pytest.raises(dsp._lib.DSPB200Error):
                check(lib.dspb200_mt_pgram_batch_exec_dev(plan.handle, *args, None))
        with pytest.raises(dsp._lib.DSPB200Error):
            check(lib.dspb200_mt_pgram_batch_exec(plan.handle, None, n, nchan, out.ptr))
        with pytest.raises(dsp._lib.DSPB200Error):                 # len != n, host form
            check(lib.dspb200_mt_pgram_batch_exec(plan.handle, s.ptr, n - 1, nchan, out.ptr))
        L = 1024
        with pytest.raises(dsp._lib.DSPB200Error):
            check(lib.dspb200_mt_spectrogram_batch_exec_dev(spec.handle, None, L, nchan, out.ptr, None))
        with pytest.raises(dsp._lib.DSPB200Error):                 # out overlaps s
            check(lib.dspb200_mt_spectrogram_batch_exec_dev(spec.handle, s.ptr, L, nchan, s.ptr, None))
        with pytest.raises(dsp._lib.DSPB200Error):                 # not a multitaper plan
            p = kp._plan(dsp, F32, 256, 128, 256, True, None)
            try:
                check(lib.dspb200_mt_spectrogram_batch_exec_dev(p.handle, s.ptr, L, nchan, out.ptr, None))
            finally:
                p.close()
        # nothing to do: no channel, no segment
        check(lib.dspb200_mt_pgram_batch_exec_dev(plan.handle, None, n, 0, None, None))
        check(lib.dspb200_mt_spectrogram_batch_exec_dev(spec.handle, s.ptr, 255, nchan, out.ptr, None))
        check(lib.dspb200_mt_spectrogram_batch_exec(spec.handle, None, L, 0, None))
        device.sync()
        assert dsp.launch_count() == n0
    finally:
        plan.close()
        spec.close()
        device.empty_cache()


@pytest.mark.gpu
def test_front_end_device_and_host_forms():
    from dspb200 import device
    rng = np.random.default_rng(11)
    S = np.asfortranarray(rng.standard_normal((4096, 5)).astype(np.float32))          # fused sizes: nfft 4096 and 512
    dS = device.to_device(S)
    ph = dsp.mt_pgram(S, nw=3)
    pd = dsp.mt_pgram(dS, nw=3)
    assert isinstance(pd.power, device.DeviceArray) and pd.power.shape == (ph.power.shape[0], 5)
    assert same_bits(pd.power.to_host(), ph.power)
    for c in (0, 4):
        assert same_bits(dsp.mt_pgram(np.ascontiguousarray(S[:, c]), nw=3).power, ph.power[:, c])
    sh = dsp.mt_spectrogram(S, 512, 384, nw=3)
    sd = dsp.mt_spectrogram(dS, 512, 384, nw=3)
    assert sh.power.shape == (257, (4096 - 512) // 128 + 1, 5)
    assert same_bits(sd.power.to_host(), sh.power)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_pgram(dS, dsp.MTConfig(np.float64, 4096, nw=3))
    with pytest.raises(dsp.DimensionMismatch):
        dsp.mt_pgram(dS, dsp.MTConfig(np.float32, 4095, nw=3))
    z = dsp.mt_spectrogram(device.to_device(np.ones((100, 2), np.float32)), 512, 384, nw=3)
    assert z.power.shape == (257, 0, 2)
