"""Multitaper cross spectra and coherence of many epochs in one call (an extension of mt_cross_power_spectra /
mt_coherence, src/multitaper.jl:551-790): `dspb200_mt_cross_spectra_epochs(_exec)`, the 3-D front ends, the `!` forms,
`MTCoherenceConfig` and `allocate_output`.

The estimate of an n_channels x n_samples x E signal is S / E with S = ((M_0 + M_1) + M_2) + ..., M_e the matrix call on
signal[:, :, e], summed in epoch order in the output eltype, real and imaginary parts each divided by E in that eltype.
The GPU tests check that bit for bit against this composition of device matrix calls, check E = 1 against the matrix call,
and check the mean against the float64 / long-double reference within the per-element bound of mt_cross_ref summed over
the epochs, plus the rounding of E - 1 running sums and one division.  Epoch groups: the raw spectra of all tapers of a
group's epochs (nout x n_channels x ntapers cx<T> per epoch) fit 1 GiB, at least one epoch per group.  At odd or
non-7-smooth cuFFT sizes a column's batched transform depends on its neighbours in the batch (Float32 nfft 1031 with three
channels differed when two epochs shared a batch), so there each epoch is transformed by a call of its own.

CPU tests run the front-end rules against a stand-in plan."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import dspb200 as dsp
from dspb200 import _lib
from dspb200 import multitaper as mtm

from test_client_kernel_paths import (F32, F64, REALS, Guarded, HostOut, _ccx, _real, coherence_interval, check_coherence,
                                      check_elems, eps, largest_prime, mt_cases, mt_cross_ref, mt_range, mt_ref, mt_signal, mt_tapers,
                                      same_bits)
from test_stft_stream import _AddressOnly

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dspb200.h")
ENTRIES = ("dspb200_mt_cross_spectra_epochs", "dspb200_mt_cross_spectra_epochs_exec")
SCRATCH = 1 << 30                       # MT_CROSS_SCRATCH (spectral.cu)
EINVALID = -1                           # DSPB200_EINVALID


def group_size(nout, nchan, ntapers, dt, nepochs):
    """Epochs per group, restated: the raw spectra of a group's epochs fit SCRATCH bytes, at least one epoch."""
    per_epoch = nout * nchan * ntapers * np.dtype(_ccx(dt)).itemsize
    return max(1, min(nepochs, SCRATCH // per_epoch))


def groups(nout, nchan, ntapers, dt, nepochs):
    g = group_size(nout, nchan, ntapers, dt, nepochs)
    return [min(g, nepochs - e0) for e0 in range(0, nepochs, g)]


def test_group_rule():
    # Float64 nfft 8192 x 64 channels x 7 tapers: 29.4 MB of spectra per epoch, 36 epochs per group
    assert group_size(4097, 64, 7, F64, 1000) == 36
    assert groups(4097, 64, 7, F64, 37) == [36, 1]
    assert groups(4097, 64, 7, F64, 80) == [36, 36, 8]
    assert groups(8193, 64, 7, F32, 37) == [36, 1]
    assert groups(129, 3, 3, F32, 17) == [17]
    assert group_size(1 << 30, 64, 7, F64, 5) == 1        # an epoch past the budget still forms a group


# =============================================================================== CPU: declarations and bindings

def test_entry_points_declared_bound_and_not_dev():
    with open(HEADER) as f:
        text = f.read()
    for name in ENTRIES:
        assert re.search(r"DSPB200_API int " + name + r"\(", text), name
        assert name in _lib.SIGNATURES and not name.endswith("_dev")
        assert hasattr(_lib.lib, name)
    assert "returns after the work on that stream has completed" in " ".join(text.split())
    for name in ("MTCoherenceConfig", "mt_cross_power_spectra_", "mt_coherence_", "allocate_output"):
        assert hasattr(dsp, name), name


# =============================================================================== CPU: front end against a stand-in plan

class _StubMtPlan:
    """Stands in for the device plan: records the cross-spectra calls and writes the epoch count into the output."""
    calls = []

    def __init__(self, dtype, n, noverlap, nfft, onesided, tapers):
        self.dtype, self.n, self.nfft = np.dtype(dtype), n, nfft
        self.nout = nfft // 2 + 1 if onesided else nfft

    def cross_spectra(self, sig, nchan, demean, f_lo, nf, coherence, out):
        _StubMtPlan.calls.append(("host", sig.shape, sig.dtype, nchan, demean, f_lo, nf, coherence, out.shape, out.dtype))
        out[...] = 1

    def cross_spectra_dev(self, ptr, nchan, demean, f_lo, nf, coherence, out_ptr):
        _StubMtPlan.calls.append(("dev", ptr, nchan, demean, f_lo, nf, coherence, out_ptr))

    def cross_spectra_epochs(self, sig, nchan, nepochs, demean, f_lo, nf, coherence, out):
        _StubMtPlan.calls.append(("host3", sig.shape, sig.dtype, nchan, nepochs, demean, f_lo, nf, coherence, out.shape,
                                  out.dtype, sig.flags.f_contiguous))
        out[...] = nepochs

    def cross_spectra_epochs_dev(self, ptr, nchan, nepochs, demean, f_lo, nf, coherence, out_ptr):
        _StubMtPlan.calls.append(("dev3", ptr, nchan, nepochs, demean, f_lo, nf, coherence, out_ptr))

    def close(self):
        pass


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(mtm._lib, "MtPlan", _StubMtPlan)
    monkeypatch.setattr(mtm, "DeviceArray", _AddressOnly)
    _StubMtPlan.calls = []
    return _StubMtPlan


def _config(dt, nchan=3, n=100, **kw):
    return dsp.MTCrossSpectraConfig(nchan, n, eltype=dt, nw=2, **kw)


@pytest.mark.parametrize("dt", REALS, ids=lambda d: d.name)
def test_shapes_and_calls(stub, dt):
    cfg = _config(dt, demean=True, freq_range=(0.1, 0.3))
    x = np.ones((3, 100, 4), dtype=dt)
    r = dsp.mt_cross_power_spectra(x, cfg)
    assert r.power.shape == (3, 3, cfg.nfreq) and r.power.dtype == _ccx(dt) and (r.power == 4).all()
    assert stub.calls[-1] == ("host3", (3, 100, 4), dt, 3, 4, True, cfg.freq_lo, cfg.nfreq, False, (3, 3, cfg.nfreq), _ccx(dt),
                              True)
    c = dsp.mt_coherence(x, cfg)
    assert c.coherence.shape == (3, 3, cfg.nfreq) and c.coherence.dtype == _real(dt)
    assert stub.calls[-1][0] == "host3" and stub.calls[-1][8] is True
    # one epoch as a 3-D array still runs the epoch entry point (one epoch gives the matrix call's bits)
    dsp.mt_cross_power_spectra(x[:, :, :1], cfg)
    assert stub.calls[-1][0] == "host3" and stub.calls[-1][4] == 1
    # keyword form: the defaults come from size(signal)[:2]
    r = dsp.mt_cross_power_spectra(np.ones((2, 64, 3), dtype=dt), nw=2)
    assert r.power.shape == (2, 2, 33) and stub.calls[-1][3:5] == (2, 3)


@pytest.mark.parametrize("dt", REALS, ids=lambda d: d.name)
def test_matrix_calls_unchanged(stub, dt):
    cfg = _config(dt, freq_range=(0.05, 0.4))
    x = np.ones((3, 100), dtype=dt)
    r = dsp.mt_cross_power_spectra(x, cfg)
    assert stub.calls == [("host", (3, 100), dt, 3, False, cfg.freq_lo, cfg.nfreq, False, (3, 3, cfg.nfreq), _ccx(dt))]
    assert r.power.shape == (3, 3, cfg.nfreq)
    d = _AddressOnly((3, 100), dt)
    out = dsp.mt_coherence(d, cfg).coherence
    assert stub.calls[-1] == ("dev", d.ptr, 3, False, cfg.freq_lo, cfg.nfreq, True, out.ptr)
    d3 = _AddressOnly((3, 100, 5), dt)
    out = dsp.mt_cross_power_spectra(d3, cfg).power
    assert isinstance(out, dsp.device.DeviceArray) and out.shape == (3, 3, cfg.nfreq) and out.dtype == _ccx(dt)
    assert stub.calls[-1] == ("dev3", d3.ptr, 3, 5, False, cfg.freq_lo, cfg.nfreq, False, out.ptr)


def test_refusals(stub):
    cfg = _config(F32)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.mt_cross_power_spectra(np.ones((3, 99, 2), F32), cfg)
    with pytest.raises(dsp.DimensionMismatch):
        dsp.mt_coherence(np.ones((4, 100, 2), F32), cfg)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_cross_power_spectra(np.ones((3, 100, 0), F32), cfg)            # n_epochs == 0
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_cross_power_spectra(_AddressOnly((3, 100, 0), F32), cfg)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_cross_power_spectra(np.ones((3, 100, 2, 1), F32), cfg)          # rank 4
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_cross_power_spectra(np.ones((3, 100, 2), np.complex64), cfg)   # complex input stays refused
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_cross_power_spectra(_AddressOnly((3, 100, 2), F64), cfg)       # device eltype must be the config's
    assert stub.calls == []


def test_residency_and_eltype_of_out(stub):
    cfg = _config(F32)
    shape = (3, 3, cfg.nfreq)
    x, d = np.ones((3, 100, 2), F32), _AddressOnly((3, 100, 2), F32)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_cross_power_spectra_(np.empty(shape, np.complex64), d, cfg)    # a device signal needs a device out
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_cross_power_spectra_(_AddressOnly(shape, np.complex64), x, cfg)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_cross_power_spectra_(np.empty(shape, np.complex128), x, cfg)   # eltype
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_coherence_(np.empty(shape, np.float64), x, dsp.MTCoherenceConfig(cfg))
    with pytest.raises(dsp.ArgumentError):                                       # out overlapping the signal
        dsp.mt_cross_power_spectra_(_AddressOnly(shape, np.complex64, _ptr=d.ptr + 8), d, cfg)
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_coherence_(np.empty(shape, np.float32), x, cfg)                 # the ! coherence takes an MTCoherenceConfig
    with pytest.raises(dsp.ArgumentError):
        dsp.mt_cross_power_spectra_(np.empty(shape, np.complex64), x, dsp.MTCoherenceConfig(cfg))
    assert stub.calls == []
    o = _AddressOnly(shape, np.complex64)
    r = dsp.mt_cross_power_spectra_(o, d, cfg)
    assert r.power is o and stub.calls[-1] == ("dev3", d.ptr, 3, 2, False, cfg.freq_lo, cfg.nfreq, False, o.ptr)


def test_bang_forms_size_checks(stub):
    # src/multitaper.jl:557-564 and :759-767: signal (n_channels, n_samples), output (n_channels, n_channels, nfreq)
    cfg = _config(F64, freq_range=(0.1, 0.2))
    ccfg = dsp.MTCoherenceConfig(cfg)
    for x in (np.ones((3, 100), F64), np.ones((3, 100, 2), F64)):
        for bad in ((3, 3, cfg.nfreq + 1), (3, 2, cfg.nfreq), (3, 3)):
            with pytest.raises(dsp.DimensionMismatch):
                dsp.mt_cross_power_spectra_(np.empty(bad, np.complex128, order="F"), x, cfg)
            with pytest.raises(dsp.DimensionMismatch):
                dsp.mt_coherence_(np.empty(bad, np.float64, order="F"), x, ccfg)
        with pytest.raises(dsp.DimensionMismatch):
            dsp.mt_cross_power_spectra_(dsp.allocate_output(cfg), x[:2], cfg)
        out = dsp.allocate_output(cfg)
        r = dsp.mt_cross_power_spectra_(out, x, cfg)
        assert r.power is out and np.array_equal(r.freq, cfg.freq)
        out = dsp.allocate_output(ccfg)
        c = dsp.mt_coherence_(out, x, ccfg)
        assert c.coherence is out and np.array_equal(c.freq, cfg.freq)
        assert stub.calls[-1][0] == ("host" if x.ndim == 2 else "host3")
    # a C-ordered out is filled through a Fortran copy
    out = np.empty((3, 3, cfg.nfreq), np.complex128, order="C")
    r = dsp.mt_cross_power_spectra_(out, np.ones((3, 100, 2), F64), cfg)
    assert r.power is out and (out == 2).all()


@pytest.mark.parametrize("dt", REALS, ids=lambda d: d.name)
def test_coherence_config_and_allocate_output(stub, dt):
    cfg = _config(dt, nchan=5, freq_range=(0.1, 0.3), demean=True)
    for ccfg in (dsp.MTCoherenceConfig(cfg), dsp.MTCoherenceConfig(5, 100, eltype=dt, nw=2, freq_range=(0.1, 0.3), demean=True),
                 dsp.MTCoherenceConfig(5, cfg.mt_config, freq_range=(0.1, 0.3), demean=True)):
        cs = ccfg.cs_config
        assert cs.n_channels == 5 and cs.demean and cs.nfreq == cfg.nfreq and np.array_equal(ccfg.freq, cfg.freq)
        a = dsp.allocate_output(ccfg)
        assert a.shape == (5, 5, cfg.nfreq) and a.dtype == _real(dt) and a.flags.f_contiguous
    assert dsp.MTCoherenceConfig(cfg).cs_config is cfg
    a = dsp.allocate_output(cfg)
    assert a.shape == (5, 5, cfg.nfreq) and a.dtype == _ccx(dt) and a.flags.f_contiguous
    with pytest.raises(dsp.ArgumentError):
        dsp.MTCoherenceConfig(cfg, 100)
    with pytest.raises(dsp.ArgumentError):
        dsp.allocate_output(cfg.mt_config)                                     # allocate_output(MTConfig) stays refused
    # mt_coherence takes either config kind; the settings are those of the cross-spectra config
    x = np.ones((5, 100, 3), dt)
    dsp.mt_coherence(x, cfg)
    first = stub.calls[-1]
    dsp.mt_coherence(x, dsp.MTCoherenceConfig(cfg))
    assert stub.calls[-1] == first and first[5:9] == (True, cfg.freq_lo, cfg.nfreq, True)


# =============================================================================== GPU helpers

def _ptr_at(g, offset_elems):
    return g.ptr + offset_elems * g.dt.itemsize


def _matrix_dev(dsp_, mt, ptr, nchan, demean, f_lo, nf, coh, odt):
    from dspb200 import device
    out = device.DeviceArray((nchan * nchan * nf,), odt)
    dsp_._lib.check(dsp_._lib.lib.dspb200_mt_cross_spectra_exec_dev(mt.handle, ptr, nchan, int(demean), f_lo, nf, int(coh),
                                                                    out.ptr, None))
    return out.to_host().reshape((nchan, nchan, nf), order="F")


def _compose(dsp_, mt, gx, nchan, n, nepochs, demean, f_lo, nf, dt):
    """The epoch mean as a host composition of device matrix calls: epoch-ordered sum in T, then parts divided by E in T."""
    S = None
    for e in range(nepochs):
        M = _matrix_dev(dsp_, mt, _ptr_at(gx, e * nchan * n), nchan, demean, f_lo, nf, False, _ccx(dt))
        S = M.copy() if S is None else S + M
    if nepochs > 1:
        E = dt.type(nepochs)
        re, im = S.real / E, S.imag / E
        assert re.dtype == dt
        S = np.empty(S.shape, _ccx(dt), order="F")
        S.real, S.imag = re, im
    return S


def _epochs_dev(dsp_, mt, ptr, nchan, nepochs, demean, f_lo, nf, coh, dt, stream=None):
    odt = _real(dt) if coh else _ccx(dt)
    go = Guarded(odt, nchan * nchan * nf)
    dsp_._lib.check(dsp_._lib.lib.dspb200_mt_cross_spectra_epochs(mt.handle, ptr, nchan, nepochs, int(demean), f_lo, nf,
                                                                  int(coh), go.ptr, stream))
    return go


def _epochs_host(dsp_, mt, x3, nchan, nepochs, demean, f_lo, nf, coh, dt):
    odt = _real(dt) if coh else _ccx(dt)
    out = HostOut(odt, nchan * nchan * nf)
    xf = np.asfortranarray(x3)
    dsp_._lib.check(dsp_._lib.lib.dspb200_mt_cross_spectra_epochs_exec(mt.handle, dsp_._lib.ptr(xf), nchan, nepochs, int(demean),
                                                                       f_lo, nf, int(coh), out.ptr))
    return out.data((nchan, nchan, nf))


def _mean_ref(x3, rows, nfft, demean, f_lo, nf, dt):
    """Reference epoch mean and its bound: per-epoch mt_cross_ref bounds summed, plus (E + 1) u sum_e (|S_e| + B_e) for the
    E - 1 running sums in T and the division, over E."""
    E = x3.shape[2]
    S = B = A = 0
    for e in range(E):
        X, cf, dA = mt_ref(x3[:, :, e], rows, nfft, demean, dt)
        Se, Be = mt_cross_ref(X, cf, dA, f_lo, nf, dt)
        S, B, A = S + Se, B + Be, A + np.abs(Se).astype(np.float64) + Be
    u = eps(dt)
    return S / E, (B + (E + 1) * u * A) / E


@pytest.fixture(scope="module")
def gdsp():
    return pytest.importorskip("dspb200")


EPOCHS = (1, 2, 3, 17)


# =============================================================================== GPU: bit for bit against the composition

@pytest.mark.gpu
@pytest.mark.parametrize("dt", REALS, ids=lambda d: d.name)
def test_epochs_against_composition(gdsp, dt):
    from dspb200 import device
    rng = np.random.default_rng([dt.num, 31])
    try:
        cases = mt_cases(dt) + [(64, 256, 256, 7, True, True, "none"), (64, 1000, 1000, 3, False, False, "interior")]
        for case in cases:
            nchan, n, nfft, nt, weighted, demean, frange = case
            rows = mt_tapers(n, nt, weighted)
            nout = nfft // 2 + 1
            f_lo, nf = mt_range(frange, nout)
            mt = gdsp._lib.MtPlan(dt, n, 0, nfft, True, rows)
            try:
                for E in EPOCHS:
                    if n * nchan * E > (1 << 22) and E > 3:
                        continue                                   # the largest transforms: E <= 3 is enough
                    x3 = np.stack([mt_signal(rng, nchan, n, dt, 1e3 if demean else 0.0) for _ in range(E)], axis=2)
                    gx = Guarded(dt, x3.size, rng, x3)
                    what = (case, E)
                    d = {coh: _epochs_dev(gdsp, mt, gx.ptr, nchan, E, demean, f_lo, nf, coh, dt) for coh in (False, True)}
                    got = {coh: d[coh].data((nchan, nchan, nf)) for coh in (False, True)}
                    gx.data()                                      # the input and its guard cells are unchanged
                    for coh in (False, True):                      # host form: bit for bit the device form
                        assert same_bits(_epochs_host(gdsp, mt, x3, nchan, E, demean, f_lo, nf, coh, dt), got[coh]), what
                    if nf == 0:
                        assert got[False].size == 0
                        continue
                    S = _compose(gdsp, mt, gx, nchan, n, E, demean, f_lo, nf, dt)
                    assert same_bits(got[False], S), what
                    if E == 1:                                     # the matrix call, both results
                        Cm = _matrix_dev(gdsp, mt, gx.ptr, nchan, demean, f_lo, nf, True, _real(dt))
                        assert same_bits(got[True], Cm), what
                    assert same_bits(got[True], got[True].transpose(1, 0, 2)), what
                    if E in (1, 3):
                        Sr, Br = _mean_ref(x3, rows, nfft, demean, f_lo, nf, dt)
                        check_elems(got[False], Sr, Br, what)
                        ref, lo, hi = coherence_interval(Sr, Br, dt)
                        check_coherence(got[True].astype(np.float64), ref, lo, hi, what)
            finally:
                mt.close()
    finally:
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,nfft,nepochs", [(F64, 8192, 37), (F64, 8192, 80), (F32, 16384, 37)],
                         ids=["f64-2groups", "f64-3groups", "f32-2groups"])
def test_epoch_groups(gdsp, dt, nfft, nepochs):
    from dspb200 import device
    nchan, nt = 64, 7
    nout = nfft // 2 + 1
    gs = groups(nout, nchan, nt, dt, nepochs)
    assert len(gs) >= 2 and (gs[-1] == 1 or len(gs) >= 3)
    rng = np.random.default_rng([dt.num, nepochs])
    rows = mt_tapers(nfft, nt, True)
    f_lo, nf = nout // 3, 40                                       # a narrow range keeps the host composition small
    x3 = (rng.standard_normal((nchan, nfft, nepochs)) + 5.0).astype(dt)
    mt = gdsp._lib.MtPlan(dt, nfft, 0, nfft, True, rows)
    try:
        gx = Guarded(dt, x3.size, rng, x3)
        before = gdsp._lib.launch_count()
        go = _epochs_dev(gdsp, mt, gx.ptr, nchan, nepochs, True, f_lo, nf, False, dt)
        launches = gdsp._lib.launch_count() - before
        assert launches == len(gs) * (2 + nt), launches            # fused size: prep, one STFT launch per taper, accumulate
        got = go.data((nchan, nchan, nf))
        gx.data()
        assert same_bits(got, _compose(gdsp, mt, gx, nchan, nfft, nepochs, True, f_lo, nf, dt))
    finally:
        mt.close()
        device.empty_cache()


# =============================================================================== GPU: launches, refusals, streams

def _stft_launches(gdsp, mt, n, cols, dt):
    from dspb200 import device
    x = device.DeviceArray((n * cols,), dt)
    y = device.DeviceArray((mt.nout * cols,), _ccx(dt))
    before = gdsp._lib.launch_count()
    gdsp._lib.check(gdsp._lib.lib.dspb200_stft_exec_dev(mt.handle, x.ptr, n, cols, C.c_double(1.0), 0, y.ptr, None))
    device.sync()
    return gdsp._lib.launch_count() - before


@pytest.mark.gpu
@pytest.mark.parametrize("dt,n,nfft", [(F32, 1024, 1024), (F64, 1000, 1000), (F32, 1031, 1031)], ids=["fused", "cufft", "odd"])
def test_launch_count_matches_header(gdsp, dt, n, nfft):
    from dspb200 import device
    rng = np.random.default_rng(5)
    nchan, nt, E = 7, 3, 5
    rows = mt_tapers(n, nt, False)
    mt = gdsp._lib.MtPlan(dt, n, 0, nfft, True, rows)
    try:
        x3 = rng.standard_normal((nchan, n, E)).astype(dt)
        gx = device.to_device(np.asfortranarray(x3).ravel(order="F"))
        # fused and even 7-smooth cuFFT sizes: one STFT call per taper over all columns; other cuFFT sizes one per taper and epoch
        per_epoch = not mt.fused and (nfft % 2 == 1 or largest_prime(nfft) > 7)
        stft = E * _stft_launches(gdsp, mt, n, nchan, dt) if per_epoch else _stft_launches(gdsp, mt, n, nchan * E, dt)
        assert stft >= 1 and per_epoch == (nfft == 1031)
        for coh in (False, True):
            before = gdsp._lib.launch_count()
            _epochs_dev(gdsp, mt, gx.ptr, nchan, E, False, 0, mt.nout, coh, dt)
            assert gdsp._lib.launch_count() - before == 1 + nt * stft + 1 + (1 if coh else 0)
        before = gdsp._lib.launch_count()                                   # the matrix call: one accumulate launch
        _matrix_dev(gdsp, mt, gx.ptr, nchan, False, 0, mt.nout, False, _ccx(dt))
        assert gdsp._lib.launch_count() - before == 1 + nt * _stft_launches(gdsp, mt, n, nchan, dt) + 1
    finally:
        mt.close()
        device.empty_cache()


@pytest.mark.gpu
def test_refusals_launch_nothing(gdsp):
    from dspb200 import device
    n, nchan = 256, 3
    mt = gdsp._lib.MtPlan(F32, n, 0, n, True, mt_tapers(n, 3, False))
    cplx = gdsp._lib.MtPlan(np.complex64, n, 0, n, False, mt_tapers(n, 3, False))
    try:
        x = device.to_device(np.ones(nchan * n * 2, F32))
        out = device.DeviceArray((nchan * nchan * 129,), np.complex64)
        lib = gdsp._lib.lib
        before = gdsp._lib.launch_count()
        bad = [(mt.handle, x.ptr, nchan, 0, 0, 0, 129, 0, out.ptr, None),                 # n_epochs == 0
               (mt.handle, x.ptr, nchan, -1, 0, 0, 129, 0, out.ptr, None),
               (mt.handle, x.ptr, nchan, 2, 0, 0, 129, 0, x.ptr + 4 * n, None),          # out overlaps the signal
               (mt.handle, x.ptr, nchan, 1 << 60, 0, 0, 129, 0, out.ptr, None),          # past DSPB200_INDEX_LIMIT
               (mt.handle, x.ptr, 0, 2, 0, 0, 129, 0, out.ptr, None),                    # no channel
               (mt.handle, x.ptr, nchan, 2, 0, 100, 30, 0, out.ptr, None),               # range past the spectrum
               (mt.handle, None, nchan, 2, 0, 0, 129, 0, out.ptr, None),
               (cplx.handle, x.ptr, nchan, 2, 0, 0, 129, 0, out.ptr, None)]              # complex plan
        for args in bad:
            assert lib.dspb200_mt_cross_spectra_epochs(*args) == EINVALID, args[2:8]
        h = np.ones(nchan * n * 2, F32)
        ho = np.empty(nchan * nchan * 129, np.complex64)
        assert lib.dspb200_mt_cross_spectra_epochs_exec(mt.handle, gdsp._lib.ptr(h), nchan, 0, 0, 0, 129, 0,
                                                        gdsp._lib.ptr(ho)) == EINVALID
        assert gdsp._lib.launch_count() == before
        assert lib.dspb200_mt_cross_spectra_epochs(mt.handle, x.ptr, nchan, 2, 0, 5, 0, 0, out.ptr, None) == 0  # nf == 0
        assert gdsp._lib.launch_count() == before
    finally:
        mt.close()
        cplx.close()
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,nfft", [(F32, 1024), (F64, 1000)], ids=["fused", "cufft"])
def test_non_blocking_stream(gdsp, dt, nfft):
    torch = pytest.importorskip("torch")
    from dspb200 import device
    rng = np.random.default_rng(9)
    nchan, nt, E = 5, 3, 4
    mt = gdsp._lib.MtPlan(dt, nfft, 0, nfft, True, mt_tapers(nfft, nt, True))
    try:
        x3 = rng.standard_normal((nchan, nfft, E)).astype(dt)
        gx = Guarded(dt, x3.size, rng, x3)
        ref = {coh: _epochs_dev(gdsp, mt, gx.ptr, nchan, E, True, 0, mt.nout, coh, dt).data() for coh in (False, True)}
        st = torch.cuda.Stream()                                        # non-blocking
        torch.cuda._sleep(1 << 22)                                       # the legacy stream is busy meanwhile
        for coh in (False, True):
            go = _epochs_dev(gdsp, mt, gx.ptr, nchan, E, True, 0, mt.nout, coh, dt, C.c_void_p(st.cuda_stream))
            assert st.query(), "the call returned before its work on the stream completed"
            assert same_bits(go.data(), ref[coh])
        torch.cuda.synchronize()
    finally:
        mt.close()
        device.empty_cache()


# =============================================================================== GPU: past 32-bit indices

@pytest.mark.gpu
def test_past_2_31_elements(gdsp):
    torch = pytest.importorskip("torch")
    from dspb200 import device
    nchan, n, E, nt = 2, 1 << 24, 65, 1                        # 2^31 + 2^25 elements, 8.6 GB; element 2^31 opens epoch 64
    total = nchan * n * E
    assert total > (1 << 31) and 4 * total > (1 << 32)
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(total, generator=g, device="cuda", dtype=torch.float32)
    rows = np.hanning(n)[None, :]
    rows = rows / np.linalg.norm(rows)
    mt = gdsp._lib.MtPlan(F32, n, 0, n, True, rows)
    try:
        f_lo, nf = 1000, 24
        out = device.DeviceArray((nchan * nchan * nf,), np.complex64)
        torch.cuda.synchronize()
        gdsp._lib.check(gdsp._lib.lib.dspb200_mt_cross_spectra_epochs(mt.handle, x.data_ptr(), nchan, E, 1, f_lo, nf, 0,
                                                                      out.ptr, None))
        got = out.to_host().reshape((nchan, nchan, nf), order="F")
        S = None
        for e in range(E):
            M = _matrix_dev(gdsp, mt, x.data_ptr() + 4 * e * nchan * n, nchan, True, f_lo, nf, False, np.complex64)
            assert np.abs(M).max() > 0
            S = M.copy() if S is None else S + M
        re, im = S.real / np.float32(E), S.imag / np.float32(E)
        assert same_bits(got.real.copy(), re) and same_bits(got.imag.copy(), im)
    finally:
        mt.close()
        del x
        torch.cuda.empty_cache()
        device.empty_cache()


# =============================================================================== GPU: front ends and the MNE golden

@pytest.mark.gpu
def test_mne_golden_as_one_epoch(goldens):
    from test_gpu_parity import TOL64, _mt_cross_case
    from conftest import relerr
    fs, n, sin_1, sin_2 = _mt_cross_case(goldens)
    signal = np.stack([sin_1, sin_2])
    ref = (goldens["csd_mt_values_re"] + 1j * goldens["csd_mt_values_im"]).reshape((512, 2, 2)).transpose(2, 1, 0)
    mt_config = dsp.dpss_config(np.float64, n, fs=fs, keep_only_large_evals=True, weight_by_evals=True)
    config = dsp.MTCrossSpectraConfig(2, mt_config, demean=True)
    r3 = dsp.mt_cross_power_spectra(signal[:, :, None], config)
    assert r3.power.shape == (2, 2, 513) and relerr(r3.power[:, :, 1:], ref) < TOL64
    assert same_bits(r3.power, dsp.mt_cross_power_spectra(signal, config).power)
    d3 = dsp.device.to_device(np.asfortranarray(signal[:, :, None]))
    assert same_bits(dsp.mt_cross_power_spectra(d3, config).power.to_host(), r3.power)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", REALS, ids=lambda d: d.name)
def test_front_ends(dt):
    rng = np.random.default_rng(3)
    nchan, n, E = 4, 500, 6
    x3 = rng.standard_normal((nchan, n, E)).astype(dt)
    cfg = dsp.MTCrossSpectraConfig(nchan, n, eltype=dt, demean=True, freq_range=(0.05, 0.3), nw=3)
    ccfg = dsp.MTCoherenceConfig(cfg)
    S = dsp.mt_cross_power_spectra(x3, cfg).power
    Ch = dsp.mt_coherence(x3, ccfg).coherence
    d3 = dsp.device.to_device(np.asfortranarray(x3))
    assert same_bits(dsp.mt_cross_power_spectra(d3, cfg).power.to_host(), S)
    assert same_bits(dsp.mt_coherence(d3, cfg).coherence.to_host(), Ch)
    out = dsp.allocate_output(cfg)
    assert dsp.mt_cross_power_spectra_(out, x3, cfg).power is out and same_bits(out, S)
    out = dsp.allocate_output(ccfg)
    assert dsp.mt_coherence_(out, x3, ccfg).coherence is out and same_bits(out, Ch)
    dout = dsp.device.DeviceArray((nchan, nchan, cfg.nfreq), _ccx(dt))
    assert dsp.mt_cross_power_spectra_(dout, d3, cfg).power is dout and same_bits(dout.to_host(), S)
    # the epoch mean against a host composition of matrix front-end calls
    acc = None
    for e in range(E):
        M = dsp.mt_cross_power_spectra(np.ascontiguousarray(x3[:, :, e]), cfg).power
        acc = M.copy() if acc is None else acc + M
    assert same_bits(S.real.copy(), acc.real / dt.type(E)) and same_bits(S.imag.copy(), acc.imag / dt.type(E))
    # the keyword form and a matrix's !-form result are unchanged
    m = np.ascontiguousarray(x3[:, :, 0])
    out = dsp.allocate_output(cfg)
    assert same_bits(dsp.mt_cross_power_spectra_(out, m, cfg).power, dsp.mt_cross_power_spectra(m, cfg).power)
    assert same_bits(dsp.mt_coherence(x3, demean=True, nw=3).coherence,
                     dsp.mt_coherence(x3, dsp.MTCrossSpectraConfig(nchan, n, eltype=dt, demean=True, nw=3)).coherence)
