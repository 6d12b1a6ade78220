"""xcorr, filtfilt, finddelay, shiftsignal and alignsignals on device-resident signals and channel matrices.

CPU: the new C entry points are declared, bound and exported; the front ends' argument rules, eltype promotion, residency
and route choice, run against a stand-in library that records every call; and a numpy restatement of the peak search's
key (|s|, -|center - i|, -i) against the reference's findall / argmin on crafted ties.
GPU: every device form against the host call -- filtfilt bit for bit, xcorr column by column (bit for bit on :direct and
:fft_overlapsave, within the convolution bound on :fft_simple, exact on integer data), finddelay / alignsignals exact on
integer data -- plus launch budgets and the asynchronous primitives on a caller's stream and under CUDA-graph capture.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT, approx, relerr

dsp = pytest.importorskip("dspb200")
clients = dsp.clients

NEW_SYMBOLS = ("dspb200_filtfilt_extend_async", "dspb200_xcorr_peak_async", "dspb200_shift_async", "dspb200_scale_div_async",
               "dspb200_conv_fft_columns", "dspb200_memcpy2d_d2d")
DTYPES = (np.float32, np.float64, np.complex64, np.complex128)


# =============================================================================== CPU

def test_new_symbols_are_declared_bound_exported_and_not_dev():
    hdr = open(os.path.join(ROOT, "include", "dspb200.h")).read()
    declared = set(re.findall(r"DSPB200_API\s+[\w\s\*]+?\b(dspb200_\w+)\s*\(", hdr))
    out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "dsp.jl_b200", "libdspb200.so")],
                         capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (dspb200_\w+)", out))
    for name in NEW_SYMBOLS:
        assert name in declared and name in dsp._lib.SIGNATURES and name in exported, name
        assert not name.endswith("_dev"), name


class FakeLib:
    """Stand-in for libdspb200: allocations hand out distinct fake addresses, every other call is recorded and succeeds."""

    def __init__(self):
        self.calls = []
        self._next = 1 << 40

    def __getattr__(self, name):
        if not name.startswith("dspb200_"):
            raise AttributeError(name)

        def call(*args):
            if name == "dspb200_malloc":
                args[0]._obj.value = self._next
                self._next += max(int(args[1]), 16) + 256
                return 0
            if name == "dspb200_memcpy_d2h":                      # device memory reads as zeros
                C.memset(args[0], 0, int(args[2]))
                return 0
            if name in ("dspb200_free", "dspb200_stream_sync", "dspb200_memcpy_h2d"):
                return 0
            self.calls.append(name)
            return 0
        return call


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(dsp._lib, "lib", lib)
    monkeypatch.setattr(dsp.device, "_POOL", {})
    monkeypatch.setattr(dsp.device, "_POOL_BYTES", [0])
    monkeypatch.setattr(dsp.dspbase, "_OS_PLANS", {})
    return lib


def _dev(shape, dt):
    return dsp.DeviceArray(shape, dt)


def test_front_end_rules_raise_before_any_call(fake):
    x32 = _dev((100, 3), np.float32)
    with pytest.raises(dsp.ArgumentError):                       # promote_type(Float64 taps, Float32 signal) != Float32
        dsp.filtfilt(np.ones(5), x32)
    with pytest.raises(dsp.ArgumentError):                       # shorter than the filter
        dsp.filtfilt(np.ones(101, np.float32), x32)
    with pytest.raises(dsp.ArgumentError):
        dsp.filtfilt(np.ones(0, np.float32), x32)
    with pytest.raises(NotImplementedError):
        dsp.filtfilt(np.ones(3, np.float32), [1.0, 0.5], x32)
    with pytest.raises(dsp.DomainError):
        dsp.shiftsignal(x32, 101)
    with pytest.raises(dsp.DomainError):
        dsp.shiftsignal(x32, [0, -101, 3])
    with pytest.raises(dsp.DimensionMismatch):
        dsp.shiftsignal(x32, [1, 2])
    with pytest.raises(dsp.DimensionMismatch):                   # :biased needs equal lengths
        dsp.xcorr(x32, np.ones(7, np.float32), scaling="biased")
    with pytest.raises(dsp.ArgumentError):
        dsp.xcorr(x32, np.ones(7, np.float32), padmode="bogus")
    with pytest.raises(dsp.ArgumentError):
        dsp.xcorr(x32, np.ones(7, np.float32), scaling="bogus")
    with pytest.raises(dsp.ArgumentError):                       # Float64 v would promote the Float32 device signal
        dsp.xcorr(x32, np.ones(7))
    with pytest.raises(dsp.ArgumentError):
        dsp.xcorr(x32, np.ones((7, 2), np.float32))
    with pytest.raises(dsp.ArgumentError):
        dsp.xcorr(x32)
    with pytest.raises(NotImplementedError):
        dsp.finddelay(_dev((100, 3), np.complex64), np.ones(7, np.complex64))
    with pytest.raises(dsp.ArgumentError):
        dsp.finddelay(x32, np.ones(7))
    with pytest.raises(dsp.ArgumentError):
        dsp.alignsignals(x32, np.ones(0, np.float32))
    assert fake.calls == []


def test_eltypes_residency_and_launch_sequence(fake):
    x = _dev((300, 4), np.float32)
    y = dsp.filtfilt(np.ones(9, np.float32), x)
    assert isinstance(y, dsp.DeviceArray) and y.shape == x.shape and y.dtype == np.float32
    assert fake.calls[0] == "dspb200_filtfilt_extend_async" and "dspb200_fir_exec_dev" in fake.calls
    assert fake.calls[-1] == "dspb200_memcpy2d_d2d"
    fake.calls.clear()
    y = dsp.filtfilt(np.ones(34, np.float32), x)                 # 67 taps: overlap-save
    assert "dspb200_os_exec_dev" in fake.calls and "dspb200_fir_exec_dev" not in fake.calls
    fake.calls.clear()
    y = dsp.filtfilt(np.ones(34, np.complex64), _dev((300, 2), np.complex64))      # complex: always the FIR kernel
    assert y.dtype == np.complex64 and "dspb200_fir_exec_dev" in fake.calls
    fake.calls.clear()
    y = dsp.filtfilt(np.ones(3) * 2.0, 2.0, _dev((50,), np.float64))
    assert isinstance(y, dsp.DeviceArray) and y.shape == (50,)
    fake.calls.clear()
    r = dsp.xcorr(_dev((40,), np.complex64), np.ones(5, np.float32))
    assert isinstance(r, dsp.DeviceArray) and r.shape == (44,) and r.dtype == np.complex64
    r = dsp.xcorr(np.ones((40, 3)), np.ones(5, np.int64))        # host matrix: staged, host result in the promoted type
    assert isinstance(r, np.ndarray) and r.shape == (44, 3) and r.dtype == np.float64
    r = dsp.xcorr(np.ones((40, 3), np.int64), np.ones(5, np.int64))
    assert r.dtype == np.int64
    fake.calls.clear()
    r = dsp.xcorr(_dev((40, 3), np.float64), np.ones(50), padmode="longest")
    assert r.shape == (99, 3) and fake.calls[0] == "dspb200_shift_async"          # the zero padding of the columns
    fake.calls.clear()
    r = dsp.xcorr(_dev((40, 3), np.float64), np.ones(40), scaling="biased")
    assert fake.calls[-1] == "dspb200_scale_div_async"
    fake.calls.clear()
    r = dsp.xcorr(np.ones((40, 3), np.int64), np.ones(40, np.int64), scaling="biased")   # rounded, then divided on the host
    assert r.dtype == np.float64 and "dspb200_scale_div_async" not in fake.calls
    fake.calls.clear()
    d = dsp.finddelay(_dev((4000, 5), np.float32), np.ones(300, np.float32))
    assert d.dtype == np.int64 and d.shape == (5,) and fake.calls[-1] == "dspb200_xcorr_peak_async"
    assert isinstance(dsp.finddelay(_dev((4000,), np.float32), np.ones(300, np.float32)), int)
    fake.calls.clear()
    a, d = dsp.alignsignals(np.zeros((4000, 2)), np.ones(300))
    assert isinstance(a, np.ndarray) and a.shape == (4000, 2) and d.shape == (2,)
    assert fake.calls[-2:] == ["dspb200_xcorr_peak_async", "dspb200_shift_async"]
    s = dsp.shiftsignal(_dev((10, 2), np.complex128), [1, -2])
    assert isinstance(s, dsp.DeviceArray) and s.dtype == np.complex128


@pytest.mark.parametrize("nu,nv", [(10, 10), (255, 256), (256, 256), (300, 5000), (5000, 300), (100000, 100000),
                                   (70000, 20), (20, 70000), (4096, 4096), (1 << 16, 1)])
def test_route_per_column_is_the_vector_calls(fake, monkeypatch, nu, nv):
    """The device path picks, per (nu, nv), the route the host vector call conv(u, reverse(conj(v))) takes."""
    host = []
    monkeypatch.setattr(dsp._lib, "conv_direct", lambda *a: host.append("direct"))
    monkeypatch.setattr(dsp._lib, "conv_fft", lambda *a: host.append("fft_simple"))

    class Plan:
        def exec(self, *a):
            host.append("fft_overlapsave")
    monkeypatch.setattr(dsp.dspbase, "_os_plan", lambda *a: Plan())
    dsp.xcorr(np.ones(nu), np.ones(nv))
    fake.calls.clear()
    dsp.xcorr(_dev((nu, 3), np.float64), np.ones(nv))
    dev = {"dspb200_conv_nd_exec_dev": "direct", "dspb200_conv_fft_columns": "fft_simple",
           "dspb200_os_exec_dev": "fft_overlapsave"}
    assert [dev[c] for c in fake.calls if c in dev] == host
    assert clients._xcorr_route(nu, nv) == host[0]


def reference_delay(s, center):
    """finddelay's host rule (src/util.jl:360-368): findall(abs.(s) .== maximum(abs.(s))), then argmin of the distance to
    the centre (first of equals); raises on a NaN (empty set), as the reference's argmin does."""
    mag = np.abs(s)
    idxs = np.flatnonzero(mag == mag.max()) + 1
    if idxs.size == 0:
        raise ValueError("argmin of an empty collection")
    return int(center - idxs[np.argmin(np.abs(center - idxs))])


def kernel_delay(s, center, reversed_=False):
    """The peak kernel's rule restated: maximise the key (|s|, -|center - i|, -i) over the samples, i 1-based, reading the
    stored column backwards when reversed_; None when the column holds a NaN."""
    col = np.asarray(s)[::-1] if reversed_ else np.asarray(s)
    best = None
    for p, v in enumerate(np.asarray(s)):
        if np.isnan(v):
            return None
        i = (len(col) - p) if reversed_ else p + 1
        key = (abs(v), -abs(center - i), -i)
        if best is None or key > best[0]:
            best = (key, i)
    return center - best[1]


@pytest.mark.parametrize("s,center", [
    ([0.0, 1.0, 0.0, 1.0, 0.0], 3),               # equal peaks, equidistant from the centre: the lower index
    ([1.0, 0.0, 0.0, 0.0, 1.0], 3),
    ([0.0] * 7, 4),                               # all zero: the centre itself, d = 0
    ([0.0] * 7, 9),                               # centre past the end: the last index
    ([-0.0, 0.0, -0.0, 0.0], 2),                  # -0.0 == 0.0: every sample ties
    ([5.0, 1.0, 2.0, 3.0], 3),                    # peak at the start
    ([1.0, 2.0, 3.0, -7.0], 1),                   # peak at the end, negative
    ([3.0, -3.0, 3.0, -3.0, 3.0, -3.0], 4),
    ([2.0, 2.0], 1), ([2.0, 2.0], 2),
])
def test_peak_key_matches_findall_argmin(s, center):
    s = np.asarray(s)
    assert kernel_delay(s, center) == reference_delay(s, center)
    # the reversed storage (xcorr(x, y) standing for xcorr(y, x)) reaches the same sample
    assert kernel_delay(s[::-1].copy(), center, reversed_=True) == reference_delay(s, center)


def test_peak_rule_nan_and_reversed_identity():
    with pytest.raises(ValueError):
        reference_delay(np.array([1.0, np.nan, 2.0]), 2)
    assert kernel_delay(np.array([1.0, np.nan, 2.0]), 2) is None
    rng = np.random.default_rng(4)
    for nx, ny in ((50, 20), (20, 50), (33, 33)):
        x, y = rng.integers(-9, 10, nx).astype(float), rng.integers(-9, 10, ny).astype(float)
        s = np.correlate(y, x, mode="full")       # xcorr(y, x)
        r = np.correlate(x, y, mode="full")       # xcorr(x, y)
        assert np.array_equal(s, r[::-1])
        assert kernel_delay(r, nx, reversed_=True) == reference_delay(s, nx)


# =============================================================================== GPU

def randn(rng, shape, dt):
    dt = np.dtype(dt)
    if dt.kind == "c":
        return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(dt)
    return rng.standard_normal(shape).astype(dt)


def randint(rng, shape, dt, lo=-8, hi=9):
    dt = np.dtype(dt)
    a = rng.integers(lo, hi, shape).astype(np.float64)
    if dt.kind == "c":
        a = a + 1j * rng.integers(lo, hi, shape)
    return a.astype(dt)


class Guarded:
    """A DeviceArray view at an odd element offset inside a larger buffer whose other cells hold a sentinel."""

    def __init__(self, host, guard=5):
        host = np.asfortranarray(host)
        self.n, self.guard = host.size, guard
        self.base = dsp.DeviceArray((host.size + 2 * guard,), host.dtype)
        self.sentinel = np.full(host.size + 2 * guard, 1234.5, dtype=host.dtype)
        self.sentinel[guard:guard + host.size] = host.ravel(order="F")
        self.base.copy_from_host(self.sentinel)
        self.arr = dsp.DeviceArray(host.shape, host.dtype, _base=self.base, _ptr=self.base.ptr + guard * host.dtype.itemsize)

    def check(self):
        assert np.array_equal(self.base.to_host(), self.sentinel, equal_nan=True), "a guard cell or the input was written"


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return (a.shape == b.shape and a.dtype == b.dtype
            and np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8)))


@pytest.mark.gpu
@pytest.mark.parametrize("nb", [1, 2, 9, 33, 34, 257, 1030])
@pytest.mark.parametrize("dt", DTYPES)
def test_filtfilt_device_is_bit_identical_to_host(dt, nb):
    rng = np.random.default_rng(nb)
    b = randn(rng, nb, dt)
    for nchan in (1, 3, 70):
        for n in (nb, 2 * nb + 1):
            x = randn(rng, (n, nchan), dt)
            g = Guarded(x if nchan > 1 else x[:, 0])
            got = dsp.filtfilt(b, g.arr)
            g.check()
            assert isinstance(got, dsp.DeviceArray) and got.shape == g.arr.shape
            got = got.to_host().reshape(n, nchan, order="F")
            for c in range(nchan):
                assert same_bits(got[:, c], dsp.filtfilt(b, x[:, c])), (dt, nb, nchan, n, c)
    if np.dtype(dt).kind == "f":                              # filtfilt(b, a, x): taps normalised by a[1] as on the host
        x = randn(rng, 3 * nb + 2, dt)
        a = np.full(1, 2, dt)
        assert same_bits(dsp.filtfilt(b * 2, a, dsp.to_device(x)).to_host(), dsp.filtfilt(b * 2, a, x))


def _cols_of(r, nchan):
    r = r.to_host() if isinstance(r, dsp.DeviceArray) else r
    return r.reshape(r.shape[0], nchan, order="F")


@pytest.mark.gpu
def test_xcorr_reference_cases_on_device():
    # test/dsp.jl:317-345 with u on the device
    D = lambda a, dt=np.float64: dsp.to_device(np.asarray(a, dtype=dt))
    h = lambda r: r.to_host()
    assert np.array_equal(h(dsp.xcorr(D([1, 2]), [3, 4])), [4, 11, 6])
    assert np.array_equal(h(dsp.xcorr(D([1, 2, 3]), [4, 5])), [5, 14, 23, 12])
    assert np.array_equal(h(dsp.xcorr(D([1, 2, 3]), [4, 5], padmode="longest")), [0, 5, 14, 23, 12])
    assert np.array_equal(h(dsp.xcorr(D([1, 2, 3]), D([4, 5]), padmode="none")), [5, 14, 23, 12])
    assert np.array_equal(h(dsp.xcorr(D([1, 2]), [3, 4, 5])), [5, 14, 11, 6])
    assert np.array_equal(h(dsp.xcorr(D([1, 2]), [3, 4, 5], padmode="longest")), [5, 14, 11, 6, 0])
    assert np.array_equal(h(dsp.xcorr(D([1.0j], np.complex128), [1.0j])), [1])
    exp = np.array([5, 14, 23, 12])
    C = np.complex128
    assert approx(h(dsp.xcorr(D(np.array([1, 2, 3]) * 1.0j, C), np.array([4, 5], dtype=C))), exp * 1j)
    assert approx(h(dsp.xcorr(D([1, 2, 3], C), np.array([4, 5]) * 1.0j)), -exp * 1j)
    assert approx(h(dsp.xcorr(D(np.array([1, 2, 3]) * 1.0j, C), np.array([4, 5]) * 1.0j)), exp.astype(C))
    assert np.array_equal(h(dsp.xcorr(D([1, 2, 3]))), [3, 8, 14, 8, 3])
    assert same_bits(h(dsp.xcorr(D([1., 2, 3]), scaling="biased")), dsp.xcorr([1., 2, 3], scaling="biased"))
    with pytest.raises(dsp.DimensionMismatch):
        dsp.xcorr(D([1, 2, 3]), [4, 5], scaling="biased")


# (nu, nv) per route: :direct (nu * nv < 2^16), :fft_overlapsave (v the shorter), :fft_simple
XCORR_ROUTES = [("direct", 200, 37), ("direct", 37, 200), ("fft_overlapsave", 20000, 129), ("fft_overlapsave", 20000, 700),
                ("fft_simple", 3000, 2500), ("fft_simple", 1000, 1000)]


@pytest.mark.gpu
@pytest.mark.parametrize("route,nu,nv", XCORR_ROUTES)
@pytest.mark.parametrize("dt", DTYPES)
def test_xcorr_matrix_columns_match_vector_calls(dt, route, nu, nv):
    assert clients._xcorr_route(nu, nv) == route
    rng = np.random.default_rng(nu + nv)
    nchan = 5
    u, v = randn(rng, (nu, nchan), dt), randn(rng, nv, dt)
    g = Guarded(u)
    got = _cols_of(dsp.xcorr(g.arr, v), nchan)
    g.check()
    host = _cols_of(dsp.xcorr(u, dsp.to_device(v)), nchan)     # host matrix, device v: the same computation
    assert same_bits(host, got)
    tol = 1e-5 if np.dtype(dt) in (np.dtype(np.float32), np.dtype(np.complex64)) else 1e-13
    for c in range(nchan):
        ref = dsp.xcorr(u[:, c], v)
        if route in ("direct", "fft_overlapsave"):
            assert same_bits(got[:, c], ref), (route, c)
        else:
            assert relerr(got[:, c], ref) < tol
    # integer data: exact on every route
    ui, vi = randint(rng, (nu, nchan), dt), randint(rng, nv, dt)
    got = _cols_of(dsp.xcorr(dsp.to_device(ui), vi), nchan)
    exact = np.stack([np.convolve(ui[:, c].astype(np.complex128), np.conj(vi.astype(np.complex128))[::-1])
                      for c in range(nchan)], axis=1)
    exact = exact if np.dtype(dt).kind == "c" else exact.real
    if route == "direct":                                     # the fma chain is exact on small integers
        assert np.array_equal(got, exact.astype(got.dtype))
    else:                                                     # transform rounding stays far below 1/2: rounds to the exact result
        assert np.abs(got - exact).max() < 0.25
        assert np.array_equal(np.rint(got.real), exact.real) and np.array_equal(np.rint(got.imag), exact.imag)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_xcorr_padmode_scaling_and_conjugation(dt):
    rng = np.random.default_rng(11)
    for nu, nv in ((60, 45), (45, 60), (3000, 2200), (2200, 3000)):
        u, v = randn(rng, (nu, 3), dt), randn(rng, nv, dt)
        got = _cols_of(dsp.xcorr(dsp.to_device(u), v, padmode="longest"), 3)
        for c in range(3):
            ref = dsp.xcorr(u[:, c], v, padmode="longest")
            assert got.shape[0] == ref.size
            if clients._xcorr_route(max(nu, nv), max(nu, nv)) == "direct":
                assert same_bits(got[:, c], ref)
            else:
                assert relerr(got[:, c], ref) < (1e-5 if np.dtype(dt).itemsize <= 8 and dt != np.float64 else 1e-13)
    for n in (40, 3000):
        u, v = randn(rng, (n, 2), dt), randn(rng, n, dt)
        got = _cols_of(dsp.xcorr(dsp.to_device(u), v, scaling="biased"), 2)
        plain = _cols_of(dsp.xcorr(dsp.to_device(u), v), 2)
        assert same_bits(got, plain / n)                      # the host's res / su, in the eltype
    if np.dtype(dt).kind == "c":                              # the second argument is conjugated
        u, v = randint(rng, (30, 2), dt), randint(rng, 7, dt)
        got = _cols_of(dsp.xcorr(dsp.to_device(u), v), 2)
        for c in range(2):
            assert np.array_equal(got[:, c], np.correlate(u[:, c], v, mode="full"))


@pytest.mark.gpu
def test_finddelay_alignsignals_reference_cases_on_device():
    # test/util.jl:125-170 with x on the device
    rng = np.random.default_rng(2)
    x = rng.standard_normal(200)
    d = 17
    xd = np.concatenate([np.zeros(d), x])
    D = dsp.to_device
    assert dsp.finddelay(D(xd), x) == d and dsp.finddelay(D(xd), -x) == d
    assert dsp.finddelay(D(x), xd) == -d and dsp.finddelay(D(-x), D(xd)) == -d
    assert np.array_equal(dsp.shiftsignal(D(x), d).to_host(), np.concatenate([np.zeros(d), x[:-d]]))
    assert np.array_equal(dsp.shiftsignal(D(x), -d).to_host(), np.concatenate([x[d:], np.zeros(d)]))
    y, s = dsp.alignsignals(D(xd), x)
    assert s == d and np.array_equal(y.to_host(), np.concatenate([x, np.zeros(d)]))
    y, s = dsp.alignsignals(D(x), xd)
    assert s == -d and np.array_equal(y.to_host(), np.concatenate([np.zeros(d), x[:-d]]))
    y, s = dsp.alignsignals(D(np.array([0.0, 0, 1, 2, 3])), [1, 2, 3])
    assert s == 2
    with pytest.raises(dsp.DomainError):
        dsp.shiftsignal(D(np.array([1.0])), -2)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", (np.float32, np.float64))
@pytest.mark.parametrize("n,ny", [(900, 300), (6000, 6000), (40000, 2000), (300, 900)])
def test_finddelay_alignsignals_many_channels_exact(dt, n, ny):
    rng = np.random.default_rng(n + ny)
    nchan = 70
    y = randint(rng, ny, dt)
    x = np.zeros((n, nchan), dt)
    for c in range(nchan):
        x[:, c] = randint(rng, n, dt)
        if c % 3 == 0:                                        # a shifted copy of y inside the channel
            s = int(rng.integers(0, max(1, n - ny)))
            x[s:s + min(ny, n - s), c] += 4 * y[:min(ny, n - s)]
    x[:, 5] = 0                                               # all-zero channel: d = 0
    g = Guarded(x)
    d = dsp.finddelay(g.arr, y)
    g.check()
    want = np.array([dsp.finddelay(x[:, c], y) for c in range(nchan)])
    assert d.dtype == np.int64 and np.array_equal(d, want)
    assert d[5] == 0
    if np.any(np.abs(want) > n):                              # shiftsignal(x, -d) refuses, as on the host
        with pytest.raises(dsp.DomainError):
            dsp.alignsignals(g.arr, dsp.to_device(y))
        return
    a, d2 = dsp.alignsignals(g.arr, dsp.to_device(y))
    assert np.array_equal(d2, want)
    a = a.to_host()
    for c in range(nchan):
        if abs(want[c]) <= n:
            assert np.array_equal(a[:, c], dsp.shiftsignal(x[:, c], -want[c]))
    assert np.array_equal(dsp.finddelay(x, y), want)          # host matrix


@pytest.mark.gpu
def test_finddelay_ties_random_delays_and_nan():
    rng = np.random.default_rng(9)
    n, nchan = 500, 70
    base = rng.integers(-5, 6, n).astype(np.float64)
    x = np.zeros((n, nchan))
    delays = rng.integers(-(n - 1), n, nchan)
    for c, dl in enumerate(delays):
        x[:, c] = dsp.shiftsignal(base, int(dl))
    got = dsp.finddelay(dsp.to_device(x), base)
    assert np.array_equal(got, [dsp.finddelay(x[:, c], base) for c in range(nchan)])
    bad = x.copy()
    bad[7, 3] = np.nan
    with pytest.raises(dsp.ArgumentError):
        dsp.finddelay(dsp.to_device(bad), base)
    with pytest.raises(dsp.ArgumentError):
        dsp.alignsignals(bad, base)


def tie_column(nx, y):
    """A column of two unit spikes whose |xcorr(y, x)| peaks twice, at center - k and center + k (k > 0, center = nx):
    the reference's findall / argmin takes the lower index, delay +k; the other choice would give -k."""
    for p in range(nx):
        for q in range(p + 1, min(nx, p + len(y) + 3)):
            x = np.zeros(nx)
            x[p] = x[q] = 1.0
            mag = np.abs(np.correlate(y, x, "full"))       # xcorr(y, x), exact on these integers
            idxs = np.flatnonzero(mag == mag.max()) + 1
            dist = np.abs(nx - idxs)
            if dist.min() > 0 and np.sum(dist == dist.min()) == 2:
                return x, int(dist.min())
    raise AssertionError("no tie column")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", (np.float32, np.float64))
@pytest.mark.parametrize("nx,y", [(9, [1.0, 2.0]), (300, [0, 0, 0, 1, 2, 0, 0]), (301, [0, 1, 2, 0, 0, 0, 0, 0, 0])])
def test_finddelay_tie_takes_the_lower_index(dt, nx, y):
    """Equal peaks equidistant from the centre reach the last rule of the key: the lower logical index.  The matrix route
    stores the correlation reversed, so taking the lower storage position instead would give the opposite delay."""
    y = np.asarray(y, dtype=dt)
    t, k = tie_column(nx, y.astype(np.float64))
    t = t.astype(dt)
    assert dsp.finddelay(t, y) == k                            # the host vector call: lower index, delay +k
    assert dsp.finddelay(dsp.to_device(t), y) == k             # device vector
    rng = np.random.default_rng(nx)
    m = np.stack([rng.integers(-3, 4, nx).astype(dt), t, np.zeros(nx, dt), t], axis=1)
    want = [dsp.finddelay(m[:, c], y) for c in range(4)]
    assert want[1] == want[3] == k and want[2] == 0
    assert np.array_equal(dsp.finddelay(dsp.to_device(m), y), want)     # device matrix
    assert np.array_equal(dsp.finddelay(m, dsp.to_device(y)), want)     # host matrix, device reference
    a, d = dsp.alignsignals(dsp.to_device(m), y)
    assert np.array_equal(d, want)
    assert np.array_equal(a.to_host()[:, 1], dsp.shiftsignal(t, -k))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_xcorr_overlap_save_with_the_longer_shared_vector(dt):
    """:fft_overlapsave where the shared vector is longer than every column (the usual finddelay shape with a long
    reference): the vector call makes the column the filter, the matrix route the shared vector, so the columns agree
    within the convolution bound, and exactly after rounding on integer data."""
    rng = np.random.default_rng(17)
    nu, nv, nchan = 300, 20000, 3
    assert clients._xcorr_route(nu, nv) == "fft_overlapsave"
    u, v = randn(rng, (nu, nchan), dt), randn(rng, nv, dt)
    got = _cols_of(dsp.xcorr(dsp.to_device(u), v), nchan)
    tol = 1e-5 if np.dtype(dt) in (np.dtype(np.float32), np.dtype(np.complex64)) else 1e-13
    for c in range(nchan):
        assert relerr(got[:, c], dsp.xcorr(u[:, c], v)) < tol
    ui, vi = randint(rng, (nu, nchan), dt, -2, 3), randint(rng, nv, dt, -2, 3)     # small: the Float32 bound stays < 1/4
    got = _cols_of(dsp.xcorr(dsp.to_device(ui), vi), nchan)
    for c in range(nchan):
        exact = np.convolve(ui[:, c].astype(np.complex128), np.conj(vi.astype(np.complex128))[::-1])
        assert np.abs(got[:, c] - exact).max() < 0.25
    if np.dtype(dt).kind == "f":                               # finddelay with the long reference: exact delays
        x = np.zeros((nu, nchan), dt)
        for c in range(nchan):
            s = int(rng.integers(0, nv - nu))
            x[:, c] = 4 * vi.real[s:s + nu] + randint(rng, nu, dt)
        want = [dsp.finddelay(x[:, c], vi.real) for c in range(nchan)]
        assert np.array_equal(dsp.finddelay(dsp.to_device(x), vi.real), want)


@pytest.mark.gpu
@pytest.mark.parametrize("ti", (np.int64, np.int32))
def test_xcorr_integer_host_matrix_matches_the_vector_calls(ti):
    """Integer host matrices: the correlation is rounded to the integer eltype first and :biased then divides in Float64,
    as xcorr(u[:, c], v) does."""
    rng = np.random.default_rng(3)
    for n in (3, 40, 3000):
        u, v = rng.integers(-9, 10, (n, 4)).astype(ti), rng.integers(-9, 10, n).astype(ti)
        for scaling in ("none", "biased"):
            got = dsp.xcorr(u, v, scaling=scaling)
            for c in range(4):
                ref = dsp.xcorr(u[:, c], v, scaling=scaling)
                assert got[:, c].dtype == ref.dtype and np.array_equal(got[:, c], ref), (n, scaling, c)
    got = dsp.xcorr(np.array([[1], [2], [3]]), np.array([1, 1, 1]), scaling="biased")
    assert np.array_equal(got[:, 0], np.array([1, 3, 6, 5, 3]) / 3)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_shiftsignal_matches_host(dt):
    rng = np.random.default_rng(5)
    n = 301
    x = randn(rng, (n, 4), dt)
    g = Guarded(x)
    for s in (0, 1, -1, n, -n, 17, -123):
        got = _cols_of(dsp.shiftsignal(g.arr, s), 4)
        for c in range(4):
            assert same_bits(got[:, c], dsp.shiftsignal(x[:, c], s))
    per = [5, -n, 0, n - 1]
    got = _cols_of(dsp.shiftsignal(g.arr, per), 4)
    for c in range(4):
        assert same_bits(got[:, c], dsp.shiftsignal(x[:, c], per[c]))
    g.check()
    v = dsp.to_device(x[:, 0].copy())
    for s in rng.integers(-n, n + 1, 6):
        assert same_bits(dsp.shiftsignal(v, int(s)).to_host(), dsp.shiftsignal(x[:, 0], int(s)))


def _launches(f):
    dsp.sync()
    k = dsp.launch_count()
    r = f()
    dsp.sync()
    return dsp.launch_count() - k, r


@pytest.mark.gpu
def test_launch_budgets():
    rng = np.random.default_rng(6)
    for nb, n in ((33, 5000), (257, 20000)):
        b = randn(rng, nb, np.float32)
        x = dsp.to_device(randn(rng, (n, 16), np.float32))
        dsp.filtfilt(b, x)                                    # plans made
        newb = np.convolve(b, b[::-1]).astype(np.float32)
        ext = dsp.DeviceArray((n + 2 * nb - 2, 16), np.float32)
        out = dsp.DeviceArray(ext.shape, np.float32)
        if newb.size > 66:
            own, _ = _launches(lambda: dsp.dspbase._os_plan(newb, None).exec_dev(ext.ptr, ext.shape[0], 16, out.ptr,
                                                                                    ext.shape[0], 0))
        else:
            p = dsp._lib.FirPlan(newb)
            own, _ = _launches(lambda: p.exec_dev(ext.ptr, ext.shape[0], 16, out.ptr, 0))
        k, _ = _launches(lambda: dsp.filtfilt(b, x))
        assert k == 1 + own, (nb, k, own)
    for nu, nv in ((200, 37), (20000, 129), (3000, 2500)):
        u = dsp.to_device(randn(rng, (nu, 24), np.float64))
        v = randn(rng, nv, np.float64)
        dsp.xcorr(u, v)
        one, _ = _launches(lambda: dsp.xcorr(dsp.to_device(randn(rng, (nu, 1), np.float64)), v))
        k, _ = _launches(lambda: dsp.xcorr(u, v))
        assert k == one, (nu, nv, k, one)                     # every channel in the launches of one
        if nu < 1000:
            continue
        y = randn(rng, nv, np.float64)
        dsp.finddelay(u, y)
        corr, _ = _launches(lambda: clients._conv_columns(u, nu, 24, y[::-1], np.dtype(np.float64)))
        k, _ = _launches(lambda: dsp.finddelay(u, y))
        assert k == corr + 1
        k, _ = _launches(lambda: dsp.alignsignals(u, y))
        assert k == corr + 2
    u = dsp.to_device(randn(rng, (3000, 4), np.float64))
    v = randn(rng, 3000, np.float64)
    plain, _ = _launches(lambda: dsp.xcorr(u, v))
    k, _ = _launches(lambda: dsp.xcorr(u, v, scaling="biased"))
    assert k == plain + 1


# ------------------------------------------------------------------ the asynchronous primitives on caller streams

@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("torch has no CUDA device")
    return t


def _primitive_cases(torch):
    """(name, inputs, output sizes, call(inputs, outputs, stream)) of every asynchronous primitive; buffers are torch
    tensors (flat, one eltype each)."""
    rng = np.random.default_rng(12)
    n, nchan, pad = 4099, 6, 40
    lib = dsp._lib
    x32 = rng.standard_normal(n * nchan).astype(np.float32)
    z64 = (rng.standard_normal(n * nchan) + 1j * rng.standard_normal(n * nchan)).astype(np.complex128)
    shifts = rng.integers(-n, n + 1, nchan).astype(np.int64)
    s = rng.standard_normal(n * nchan)
    s[[7, n + 100]] = 50.0
    return [
        ("extend-f32", [x32], [((n + 2 * pad) * nchan, np.float32)],
         lambda i, o, st: lib.filtfilt_extend_async(np.float32, i[0], n, nchan, pad, o[0], st)),
        ("extend-c64", [z64], [((n + 2 * pad) * nchan, np.complex128)],
         lambda i, o, st: lib.filtfilt_extend_async(np.complex128, i[0], n, nchan, pad, o[0], st)),
        ("peak-f64", [s], [(nchan, np.int64), (nchan, np.int32)],
         lambda i, o, st: lib.xcorr_peak_async(np.float64, i[0], n, nchan, n // 2, True, o[0], o[1], st)),
        ("shift-c64", [z64, shifts], [(n * nchan, np.complex128)],
         lambda i, o, st: lib.shift_async(np.complex128, i[0], n, nchan, 0, i[1], True, o[0], n, st)),
        ("shift-f32-scalar", [x32], [(n * nchan, np.float32)],
         lambda i, o, st: lib.shift_async(np.float32, i[0], n, nchan, -77, None, False, o[0], n, st)),
        ("scale-div-c64", [z64], [],
         lambda i, o, st: lib.scale_div_async(np.complex128, i[0], n * nchan, 7.0, st)),
    ]


_TORCH_DT = {np.dtype(np.float32): "float32", np.dtype(np.float64): "float64", np.dtype(np.complex64): "complex64",
             np.dtype(np.complex128): "complex128", np.dtype(np.int64): "int64", np.dtype(np.int32): "int32"}


def _tensor(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _run(torch, case, st, before=None):
    """Inputs and outputs as fresh tensors, the call on st (a torch stream or None), the results as numpy (scale-div
    writes its input in place, so the inputs are returned too)."""
    _, ins, outs, call = case
    ti = [_tensor(torch, a) for a in ins]
    to = [torch.full((m,), -3, dtype=getattr(torch, _TORCH_DT[np.dtype(d)]), device="cuda") for m, d in outs]
    torch.cuda.synchronize()
    if st is None:
        call([t.data_ptr() for t in ti], [t.data_ptr() for t in to], None)
        torch.cuda.synchronize()
    else:
        with torch.cuda.stream(st):
            if before is not None:
                before()
            call([t.data_ptr() for t in ti], [t.data_ptr() for t in to], st.cuda_stream)
        idle = st.query()
        st.synchronize()
        assert not idle, f"{case[0]}: the stream was idle when the call returned"
    return [t.cpu().numpy() for t in to + ti]


@pytest.mark.gpu
def test_async_primitives_on_a_stream_behind_a_delay_and_in_graphs(torch):
    for case in _primitive_cases(torch):
        ref = _run(torch, case, None)
        st = torch.cuda.Stream()
        got = _run(torch, case, st, before=lambda: torch.cuda._sleep(50_000_000))
        assert all(same_bits(a, b) for a, b in zip(got, ref)), case[0]
        # capture on a non-blocking stream, replay on new inputs
        _, ins, outs, call = case
        ti = [_tensor(torch, a) for a in ins]
        to = [torch.zeros((m,), dtype=getattr(torch, _TORCH_DT[np.dtype(d)]), device="cuda") for m, d in outs]
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        cs = torch.cuda.Stream()
        with torch.cuda.graph(g, stream=cs):
            call([t.data_ptr() for t in ti], [t.data_ptr() for t in to], cs.cuda_stream)
        for t, a in zip(ti, ins):
            t.copy_(_tensor(torch, a))
        for t in to:
            t.fill_(-3)
        g.replay()
        torch.cuda.synchronize()
        got = [t.cpu().numpy() for t in to + ti]
        assert all(same_bits(a, b) for a, b in zip(got, ref)), case[0] + " (graph)"
