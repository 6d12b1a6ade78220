"""lpc, arburg and levinson (src/lpc.jl) on vectors, channel matrices and device-resident signals.

CPU: a literal Float64 / Complex128 restatement of src/lpc.jl (the oracle) against the reference's test/lpc.jl; the new C
entry points declared, bound, exported and not `_dev`; the front ends' argument rules, promotion, residency, shapes and
launch counts against a stand-in library that records every call.
GPU: the device bit for bit against a restatement of the kernels' arithmetic (src/lpc.jl in the input's eltype with the
reduction order of include/dspb200.h), for all four eltypes and both methods; every Burg path on the same columns; column
independence; accuracy against the oracle; crafted columns; guard cells, caller streams, graph capture and a call past
element 2^31.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
from scipy import signal as sps

from conftest import ROOT

dsp = pytest.importorskip("dspb200")
from oracle.dspbase import fma_f32, fma_f64  # noqa: E402

NEW_SYMBOLS = ("dspb200_lpc_work_bytes", "dspb200_lpc_burg_async", "dspb200_lpc_levinson_async", "dspb200_levinson_async")
DTYPES = (np.float32, np.float64, np.complex64, np.complex128)


def _real(T):
    return np.dtype(np.float32) if np.dtype(T) in (np.float32, np.complex64) else np.dtype(np.float64)


# =============================================================================== oracle: src/lpc.jl in Float64 / Complex128

def oracle_arburg(x, p):
    """arburg, src/lpc.jl:53-92, literally, in Float64 or Complex128 (numpy's dot order)."""
    x = np.asarray(x)
    F = np.complex128 if np.iscomplexobj(x) else np.float64
    x = x.astype(F)
    n = x.size
    unnormed = abs(np.vdot(x, x))
    err = unnormed / n
    ef, eb = x.copy(), x.copy()
    a = np.zeros(p + 1, F)
    a[0] = 1
    refl = np.zeros(p, F)
    den, ratio = 2 * unnormed, 1.0
    for m in range(1, p + 1):
        cf, cb = ef[-1], eb[0]
        ef, eb = ef[:-1], eb[1:]
        den = ratio * den - (abs(cf) ** 2 + abs(cb) ** 2)
        k = -2 * np.vdot(eb, ef) / den
        refl[m - 1] = k
        rev = a[m - 1::-1][:m].copy()
        a[1:m + 1] = k * np.conj(rev) + a[1:m + 1]
        ef, eb = k * eb + ef, np.conj(k) * ef + eb
        ratio = 1 - abs(k) ** 2
        err *= ratio
    return np.conj(a), err, refl


def oracle_levinson(r, p):
    """levinson, src/lpc.jl:122-146, in Float64 or Complex128."""
    r = np.asarray(r)
    r = r.astype(np.complex128 if np.iscomplexobj(r) else np.float64)
    k = -r[1] / r[0]
    err = np.real(r[0] * (1 - abs(k) ** 2))
    a = np.zeros(p, r.dtype)
    refl = np.zeros(p, r.dtype)
    a[0] = refl[0] = k
    for m in range(2, p + 1):
        rev = a[m - 2::-1][:m - 1].copy()
        k = -(r[m] + np.sum(r[1:m] * rev)) / err
        a[:m - 1] = k * np.conj(rev) + a[:m - 1]
        a[m - 1] = refl[m - 1] = k
        err *= 1 - abs(k) ** 2
    return a, err, refl


def oracle_lpc(x, p, method="burg"):
    if method == "burg":
        a, err, _ = oracle_arburg(x, p)
        return a[1:], err
    x = np.asarray(x)
    x = x.astype(np.complex128 if np.iscomplexobj(x) else np.float64)
    n = x.size
    r = np.correlate(x, x, mode="full")[n - 1:] / n           # xcorr(x; scaling=:biased)[length(x):end]
    return oracle_levinson(r, p)[:2]


# =============================================================================== the kernels' arithmetic, restated

def fma64(a, b, c):
    """Exact Float64 fma on the whole domain the kernels meet: the oracle's fma_f64 where it is valid; a*b + c where a*b
    is exact (a zero factor, so signed zeros come out as the hardware's) or an operand is not finite; +0 for an exact
    cancellation, as round-to-nearest gives."""
    a, b, c = np.broadcast_arrays(*(np.asarray(v, dtype=np.float64) for v in (a, b, c)))
    with np.errstate(all="ignore"):
        plain = a * b + c
        r = fma_f64(np.where(np.isfinite(plain), a, 1.0), np.where(np.isfinite(plain), b, 1.0), np.where(np.isfinite(plain), c, 1.0))
    r = np.where(r == 0, 0.0, r)
    return np.where((a == 0) | (b == 0) | ~np.isfinite(a) | ~np.isfinite(b) | ~np.isfinite(c), plain, r)


def _fma(R):
    return fma_f32 if np.dtype(R) == np.float32 else fma64


def muladd(a, b, c, T):
    """muladd in eltype T: one fma for reals, Base.muladd's form for complex."""
    T = np.dtype(T)
    R = _real(T)
    f = _fma(R)
    if T.kind != "c":
        return np.asarray(f(a, b, c)).astype(T)
    z, w, x = (np.asarray(v, dtype=T) for v in (a, b, c))
    out = np.empty(np.broadcast(z, w, x).shape, T)
    out.real = f(z.real, w.real, -np.asarray(f(z.imag, w.imag, -x.real)))
    out.imag = f(z.real, w.imag, f(z.imag, w.real, x.imag))
    return out


def ordered_reduce(L, T, step):
    """The fixed reduction order of include/dspb200.h over indices 0 .. L-1: step(acc, i) is one lane's muladd for the
    index array i.  Returns a scalar of eltype T."""
    T = np.dtype(T)
    if L == 0:
        return T.type(0)
    nt = -(-L // 1024)
    base = np.arange(nt)[:, None] * 1024 + np.arange(256)[None, :]
    acc = np.zeros((nt, 256), T)
    for j in range(4):
        i = base + 256 * j
        m = i < L
        acc = np.where(m, step(acc, np.where(m, i, 0)).astype(T), acc)
    w = acc.reshape(nt, 8, 32)
    for h in (16, 8, 4, 2, 1):
        w[..., :h] = w[..., :h] + w[..., h:2 * h]
    w = w[..., 0]
    s = ((w[:, 0] + w[:, 4]) + (w[:, 2] + w[:, 6])) + ((w[:, 1] + w[:, 5]) + (w[:, 3] + w[:, 7]))
    while s.size > 1:
        h = s.size // 2
        nxt = s[0:2 * h:2] + s[1:2 * h:2]
        s = np.concatenate([nxt, s[-1:]]) if s.size % 2 else nxt
    return T.type(s[0])


def _abs2(z, R):
    if np.iscomplexobj(z):
        return R.type(R.type(z.real * z.real) + R.type(z.imag * z.imag))
    return R.type(z * z)


def _div_real(z, r, T):
    if np.dtype(T).kind == "c":
        out = np.empty((), T)
        out.real, out.imag = z.real / r, z.imag / r
        return T.type(out[()])
    return T.type(z / r)


def _smith(a, b, T):
    """Smith's complex division, as Julia's generic /(::Complex{T}, ::Complex{T}) (finite denominators)."""
    R = _real(T).type
    are, aim, bre, bim = R(a.real), R(a.imag), R(b.real), R(b.imag)
    if abs(bre) <= abs(bim):
        r = bre / bim
        den = bim + r * bre
        re, im = (are * r + aim) / den, (aim * r - are) / den
    else:
        r = bim / bre
        den = bre + r * bim
        re, im = (are + aim * r) / den, (aim - are * r) / den
    out = np.empty((), T)
    out.real, out.imag = re, im
    return T.type(out[()])


def exact_arburg(x, p):
    """arburg in x's eltype with the device's reductions: what the kernels must produce bit for bit."""
    x = np.asarray(x)
    T = x.dtype
    R = _real(T)
    cplx = T.kind == "c"
    f = _fma(R)
    n = x.size
    if cplx:
        dxx = ordered_reduce(n, R, lambda acc, i: f(x.imag[i], x.imag[i], f(x.real[i], x.real[i], acc)))
    else:
        dxx = ordered_reduce(n, R, lambda acc, i: f(x[i], x[i], acc))
    un = R.type(abs(dxx))
    err = R.type(un / R.type(n))
    den = R.type(R.type(2) * un)
    ratio = R.type(1)
    ef, eb = x.copy(), x.copy()
    a = np.zeros(p + 1, T)
    a[0] = 1
    refl = np.zeros(p, T)
    for m in range(1, p + 1):
        cf, cb = ef[n - m], eb[m - 1]
        L = n - m
        u, v = np.conj(eb[m:m + L]), ef[:L].copy()
        d = ordered_reduce(L, T, lambda acc, i: muladd(u[i], v[i], acc, T))
        den = R.type(f(ratio, den, -R.type(_abs2(cf, R) + _abs2(cb, R)))[()])
        k = _div_real(_m2(d, T) if cplx else R.type(R.type(-2) * d), den, T)      # -2 * dot(eb, ef) / den
        refl[m - 1] = k
        ao = a.copy()
        j = np.arange(1, m + 1)
        a[j] = muladd(np.full(m, k, T), np.conj(ao[m - j]), ao[j], T)
        efo, ebo = ef[:L].copy(), eb[m:m + L].copy()
        ef[:L] = muladd(np.full(L, k, T), ebo, efo, T)
        eb[m:m + L] = muladd(np.full(L, np.conj(k), T), efo, ebo, T)
        ratio = R.type(R.type(1) - _abs2(k, R))
        err = R.type(err * ratio)
    return np.conj(a), err, refl


def _m2(d, T):
    out = np.empty((), T)
    R = _real(T).type
    out.real, out.imag = R(-2) * R(d.real), R(-2) * R(d.imag)
    return T.type(out[()])


def exact_levinson(r, p):
    r = np.asarray(r)
    T = r.dtype
    R = _real(T)
    cplx = T.kind == "c"
    k = _smith(-r[1], r[0], T) if cplx else T.type(-r[1] / r[0])
    c = R.type(R.type(1) - _abs2(k, R))
    err = R.type(R.type(r[0].real * c) - R.type(r[0].imag * R.type(0))) if cplx else R.type(r[0] * c)
    a = np.zeros(p, T)
    refl = np.zeros(p, T)
    a[0] = refl[0] = k
    for m in range(2, p + 1):
        d = np.zeros((), T)
        for i in range(m - 1):
            d = muladd(r[1 + i], a[m - 2 - i], d, T)
        num = T.type(r[m] + T.type(d[()] if np.ndim(d) == 0 else d))
        k = _div_real(-num, err, T)
        ao = a.copy()
        j = np.arange(m - 1)
        a[j] = muladd(np.full(m - 1, k, T), np.conj(ao[m - 2 - j]), ao[j], T)
        a[m - 1] = refl[m - 1] = k
        err = R.type(err * R.type(R.type(1) - _abs2(k, R)))
    return a, err, refl


def exact_acf(x, p):
    x = np.asarray(x)
    T = x.dtype
    R = _real(T)
    n = x.size
    r = np.zeros(p + 1, T)
    for k in range(p + 1):
        r[k] = ordered_reduce(n - k, T, lambda acc, i: muladd(x[i + k], np.conj(x[i]), acc, T))
    if T.kind == "c":
        scl = R.type(R.type(1) / R.type(n))
        out = np.empty(p + 1, T)
        out.real = (r.real + r.imag * R.type(0)) * scl
        out.imag = (r.imag - r.real * R.type(0)) * scl
        return out
    return (r / R.type(n)).astype(T)


def exact_lpc(x, p, method):
    if method == "burg":
        a, err, _ = exact_arburg(x, p)
        return a[1:], err
    a, err, _ = exact_levinson(exact_acf(x, p), p)
    return a, err


# =============================================================================== CPU: oracle vs the reference's tests

def _ar3(T, n=50_000, seed=0):
    """test/lpc.jl: randn(T, 50000) through filt(1, coeffs, s), analysed from sample 1000 on (seeded here)."""
    rng = np.random.default_rng(seed)
    cplx = np.dtype(T).kind == "c"
    coefs = np.array([1, 0.5 + 0.2j, 0.3 - 0.5j, 0.2]) if cplx else np.array([1, 0.5, 0.3, 0.2])
    s = rng.standard_normal(n)
    if cplx:
        s = (s + 1j * rng.standard_normal(n)) / np.sqrt(2)           # randn(ComplexF64): unit variance
    x = sps.lfilter([1.0], coefs, s)[999:]
    return np.ascontiguousarray(x.astype(T)), coefs[1:], s


@pytest.mark.parametrize("T", [np.float64, np.complex128])
@pytest.mark.parametrize("method", ["burg", "levinson"])
def test_oracle_recovers_ar3(T, method):
    x, coefs, s = _ar3(T)
    a, err = oracle_lpc(x, 3, method)
    assert np.max(np.abs(a - coefs)) < 0.01
    assert abs(err - np.std(s)) / np.std(s) < 0.01                        # isapprox(e, std(s); rtol=0.01)


def test_oracle_levinson_of_complex_ramp_and_burg_default():
    a, _, _ = oracle_levinson(np.arange(1, 11) + 0j, 3)
    assert np.allclose(a.real, -np.array([1.25, 0, 0.25]))
    v = np.random.default_rng(1).random(1000)
    assert all(np.array_equal(u, w) for u, w in zip(oracle_lpc(v, 20), oracle_lpc(v, 20, "burg")))


def test_restatement_matches_oracle_on_random_data():
    rng = np.random.default_rng(3)
    for T in DTYPES:
        x = rng.standard_normal(300)
        if np.dtype(T).kind == "c":
            x = x + 1j * rng.standard_normal(300)
        x = x.astype(T)
        tol = 1e-3 if _real(T) == np.float32 else 1e-10
        for method in ("burg", "levinson"):
            a, err = exact_lpc(x, 8, method)
            ar, er = oracle_lpc(x, 8, method)
            assert np.max(np.abs(a - ar)) < tol and abs(err - er) / er < tol, (T, method)


def test_reduction_order_is_the_documented_tree():
    """Integers summed exactly in any order: the restated tree must add every index once; and -0 terms stay -0 only where
    a lane holds no +0 (the tree carries odd tiles rather than padding them)."""
    for L in (1, 2, 255, 256, 1023, 1024, 1025, 3 * 1024 + 5, 5 * 1024):
        v = np.arange(L, dtype=np.float64)
        assert ordered_reduce(L, np.float64, lambda acc, i: fma_f64(v[i], 1.0, acc)) == v.sum()
    assert ordered_reduce(0, np.float32, None) == 0


# =============================================================================== CPU: symbols and front-end rules

def test_new_symbols_are_declared_bound_exported_and_not_dev():
    hdr = open(os.path.join(ROOT, "include", "dspb200.h")).read()
    declared = set(re.findall(r"DSPB200_API\s+[\w\s\*]+?\b(dspb200_\w+)\s*\(", hdr))
    out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "dsp.jl_b200", "libdspb200.so")],
                         capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (dspb200_\w+)", out))
    for name in NEW_SYMBOLS:
        assert name in declared and name in dsp._lib.SIGNATURES and name in exported, name
        assert not name.endswith("_dev"), name
    for name in ("lpc", "arburg", "levinson", "LPCBurg", "LPCLevinson", "LPC_P_MAX", "BoundsError"):
        assert hasattr(dsp, name), name
    assert issubclass(dsp.BoundsError, IndexError)


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
            if name == "dspb200_memcpy_d2h":
                C.memset(args[0], 0, int(args[2]))
                return 0
            if name in ("dspb200_free", "dspb200_stream_sync", "dspb200_memcpy_h2d"):
                return 0
            self.calls.append((name, args))
            return 0
        return call


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(dsp._lib, "lib", lib)
    monkeypatch.setattr(dsp.device, "_POOL", {})
    monkeypatch.setattr(dsp.device, "_POOL_BYTES", [0])
    return lib


def _names(lib):
    return [c[0] for c in lib.calls if c[0] != "dspb200_lpc_work_bytes"]


def test_front_end_rules_raise_before_any_call(fake):
    x = dsp.DeviceArray((100, 3), np.float32)
    with pytest.raises(dsp.ArgumentError):
        dsp.arburg(x, 101)
    with pytest.raises(dsp.ArgumentError):
        dsp.lpc(x, -1)
    with pytest.raises(dsp.BoundsError):
        dsp.lpc(x, 100, dsp.LPCLevinson())
    with pytest.raises(dsp.BoundsError):
        dsp.lpc(x, 0, dsp.LPCLevinson())
    with pytest.raises(dsp.BoundsError):
        dsp.levinson(np.ones(4), 4)
    with pytest.raises(IndexError):
        dsp.levinson(np.ones(4), 0)
    with pytest.raises(NotImplementedError):
        dsp.arburg(np.ones(2000), 1025)
    with pytest.raises(NotImplementedError):
        dsp.lpc(np.ones(2000), 1025, dsp.LPCLevinson())
    with pytest.raises(dsp.ArgumentError):
        dsp.lpc(x, 2.0)
    with pytest.raises(dsp.ArgumentError):
        dsp.lpc(np.ones((2, 2, 2)), 1)
    with pytest.raises(dsp.ArgumentError):
        dsp.lpc(x, 2, "burg")
    assert _names(fake) == []


def test_launch_counts_shapes_and_eltypes(fake):
    for T in DTYPES:
        R = _real(T)
        x = dsp.DeviceArray((64, 5), T)
        fake.calls.clear()
        a, err, refl = dsp.arburg(x, 4)
        assert _names(fake) == ["dspb200_lpc_burg_async"]
        assert isinstance(a, dsp.DeviceArray) and a.shape == (5, 5) and a.dtype == T
        assert err.shape == (5,) and err.dtype == R and refl.shape == (4, 5) and refl.dtype == T
        fake.calls.clear()
        a, err = dsp.lpc(x, 4)
        assert _names(fake) == ["dspb200_lpc_burg_async", "dspb200_memcpy2d_d2d"] and a.shape == (4, 5)
        fake.calls.clear()
        a, err = dsp.lpc(x, 4, dsp.LPCLevinson())
        assert _names(fake) == ["dspb200_lpc_levinson_async"] and a.shape == (4, 5) and err.dtype == R
        fake.calls.clear()
        a, err, refl = dsp.levinson(x, 4)
        assert _names(fake) == ["dspb200_levinson_async"] and a.shape == (4, 5) and refl.shape == (4, 5)
        # a device vector gives device vectors and a 0-d err, with no copy
        v = dsp.DeviceArray((64,), T)
        fake.calls.clear()
        a, err = dsp.lpc(v, 4)
        assert _names(fake) == ["dspb200_lpc_burg_async"] and a.shape == (4,) and err.shape == ()
    # host inputs: integers promote, results come back on the host
    fake.calls.clear()
    a, err = dsp.lpc(np.arange(10), 3)
    assert isinstance(a, np.ndarray) and a.dtype == np.float64 and a.shape == (3,) and np.ndim(err) == 0
    assert fake.calls[-1][0] == "dspb200_lpc_burg_async" and fake.calls[-1][1][0] == 1
    a, err, refl = dsp.levinson(np.arange(1, 11) + 0j, 3)
    assert a.dtype == np.complex128 and refl.shape == (3,)
    a, err = dsp.lpc(np.ones((32, 4), np.complex64), 2, dsp.LPCLevinson())
    assert a.dtype == np.complex64 and a.shape == (2, 4) and err.dtype == np.float32 and err.shape == (4,)
    # no channels: nothing launched
    fake.calls.clear()
    a, err = dsp.lpc(dsp.DeviceArray((64, 0), np.float32), 3)
    a, err = dsp.lpc(np.ones((64, 0)), 3, dsp.LPCLevinson())
    assert _names(fake) == []


# =============================================================================== GPU

def _data(T, n, ncols, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, ncols))
    if np.dtype(T).kind == "c":
        x = x + 1j * rng.standard_normal((n, ncols))
    x = sps.lfilter([1.0], [1, 0.2, -0.3, 0.1], x, axis=0)
    return np.asfortranarray(x.astype(T))


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind == "c":
        return same_bits(a.real.copy(), b.real.copy()) and same_bits(a.imag.copy(), b.imag.copy())
    ia, ib = a.view(np.int32 if a.itemsize == 4 else np.int64), b.view(np.int32 if b.itemsize == 4 else np.int64)
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.all((ia == ib) | nan))


NS = (1, 2, 255, 1023, 1024, 1025, 4097)
PS = (0, 1, 2, 16, 32)


@pytest.mark.gpu
@pytest.mark.parametrize("T", DTYPES)
def test_device_equals_restated_kernels_bit_for_bit(T):
    for n in NS:
        x = _data(T, n, 2, n)
        for p in PS:
            if p <= n:
                a, err, refl = dsp.arburg(x, p)
                for c in range(2):
                    ea, ee, er = exact_arburg(x[:, c], p)
                    assert same_bits(a[:, c], ea) and same_bits(err[c], ee) and same_bits(refl[:, c], er), (n, p, c)
            if 1 <= p <= n - 1:
                a, err = dsp.lpc(x, p, dsp.LPCLevinson())
                for c in range(2):
                    ea, ee = exact_lpc(x[:, c], p, "levinson")
                    assert same_bits(a[:, c], ea) and same_bits(err[c], ee), ("levinson", n, p, c)
                r = np.asfortranarray(np.stack([exact_acf(x[:, c], p) for c in range(2)], axis=1))
                a, err, refl = dsp.levinson(r, p)
                for c in range(2):
                    ea, ee, er = exact_levinson(r[:, c], p)
                    assert same_bits(a[:, c], ea) and same_bits(err[c], ee) and same_bits(refl[:, c], er)


def _burg_pinned(x, p, pin):
    T = x.dtype
    n, ncols = x.shape
    xd = dsp.to_device(x)
    a = dsp.DeviceArray((p + 1, ncols), T)
    err = dsp.DeviceArray((ncols,), _real(T))
    refl = dsp.DeviceArray((p, ncols), T)
    wb = dsp._lib.lpc_work_bytes(T, n, ncols, p, 0, pin)
    work = dsp.clients._DevWords(wb, np.uint8) if wb else None
    dsp._lib.lpc_burg_async(T, xd.ptr, n, ncols, p, a.ptr, err.ptr, refl.ptr, work.ptr if work else None, pin)
    return a.to_host(), err.to_host(), refl.to_host()


@pytest.mark.gpu
@pytest.mark.parametrize("T", DTYPES)
def test_every_burg_path_gives_the_same_bits(T):
    for n in (1, 255, 1025, 4097, 70_000):
        x = _data(T, n, 3, 7 + n)
        p = min(n, 16)
        ref = _burg_pinned(x, p, 0)
        pins = [1, 2, 8] + ([-1] if 4 * n * np.dtype(T).itemsize <= 192 << 10 else [])
        for pin in pins:
            got = _burg_pinned(x, p, pin)
            assert all(same_bits(g, r) for g, r in zip(got, ref)), (n, pin)
        if n <= 4097:
            ea, ee, er = exact_arburg(x[:, 1], p)
            assert same_bits(ref[0][:, 1], ea) and same_bits(ref[1][1], ee)


@pytest.mark.gpu
@pytest.mark.parametrize("T", DTYPES)
def test_columns_are_independent(T):
    x = _data(T, 300, 70, 11)
    for method in (dsp.LPCBurg(), dsp.LPCLevinson()):
        a, err = dsp.lpc(x, 12, method)
        for c in (0, 33, 69):
            av, ev = dsp.lpc(x[:, c].copy(), 12, method)
            assert same_bits(a[:, c], av) and same_bits(err[c], ev)
        perm = np.asfortranarray(x[:, [5, 5, 69, 0, 5]])
        ap, ep = dsp.lpc(perm, 12, method)
        assert same_bits(ap, a[:, [5, 5, 69, 0, 5]]) and same_bits(ep, err[[5, 5, 69, 0, 5]])
        ad, ed = dsp.lpc(dsp.to_device(x), 12, method)
        assert same_bits(ad.to_host(), a) and same_bits(ed.to_host(), err)
        for nc in (1, 3):
            a1, e1 = dsp.lpc(np.asfortranarray(x[:, :nc]), 12, method)
            assert same_bits(a1, a[:, :nc]) and same_bits(e1, err[:nc])


@pytest.mark.gpu
def test_seventy_thousand_channels():
    x = _data(np.float32, 64, 70_000, 5)
    for method in (dsp.LPCBurg(), dsp.LPCLevinson()):
        a, err = dsp.lpc(x, 8, method)
        for c in (0, 65_535, 65_536, 69_999):
            av, ev = dsp.lpc(x[:, c].copy(), 8, method)
            assert same_bits(a[:, c], av) and same_bits(err[c], ev), c


@pytest.mark.gpu
@pytest.mark.parametrize("T", DTYPES)
def test_reference_ar3_and_accuracy_against_the_oracle(T):
    x, coefs, s = _ar3(T)
    for method in ("burg", "levinson"):
        a, err = dsp.lpc(x, 3, dsp.LPCBurg() if method == "burg" else dsp.LPCLevinson())
        assert np.max(np.abs(a - coefs)) < 0.01 and abs(err - np.std(s)) / np.std(s) < 0.01
    v = np.random.default_rng(1).random(1000).astype(T)
    assert all(same_bits(u, w) for u, w in zip(dsp.lpc(v, 20), dsp.lpc(v, 20, dsp.LPCBurg())))
    assert np.allclose(dsp.levinson(np.arange(1, 11) + 0j, 3)[0].real, -np.array([1.25, 0, 0.25]))
    # accuracy: |a - a_oracle| <= 10 p n eps max(1, |a_oracle|), a deliberately loose linear bound in n and p
    eps = np.finfo(_real(T)).eps
    for n, p in ((1024, 16), (4097, 32)):
        x = _data(T, n, 1, n)[:, 0]
        for method in ("burg", "levinson"):
            a, err = dsp.lpc(x, p, dsp.LPCBurg() if method == "burg" else dsp.LPCLevinson())
            ar, er = oracle_lpc(x, p, method)
            bound = 10 * p * n * eps * max(1.0, np.max(np.abs(ar)))
            ratio = np.max(np.abs(a - ar)) / bound
            print(f"{np.dtype(T).name} {method} n={n} p={p}: error / bound = {ratio:.2e}")
            assert ratio <= 1 and abs(err - er) <= bound * er


@pytest.mark.gpu
@pytest.mark.parametrize("T", DTYPES)
def test_crafted_columns(T):
    n = 40
    imp = np.zeros(n, T)
    imp[0] = 3
    const = np.full(n, 2, T)
    alt = (2 * (-1.0) ** np.arange(n)).astype(T)
    cols = np.asfortranarray(np.stack([imp, const, alt], axis=1))
    a, err, refl = dsp.arburg(cols, 5)
    for c in range(3):
        ea, ee, er = exact_arburg(cols[:, c], 5)
        assert same_bits(a[:, c], ea) and same_bits(err[c], ee) and same_bits(refl[:, c], er), c
    R = _real(T)
    rr = refl.real.astype(R)
    assert np.all(rr[:, 0] == 0) and np.all(np.signbit(rr[:, 0]))               # impulse: every k is -0.0
    assert rr[0, 1] == -1 and np.all(np.isnan(rr[1:, 1]))                        # constant: k = -1, then NaN
    assert rr[0, 2] == 1 and np.all(np.isnan(rr[1:, 2]))                         # alternating: k = +1, then NaN
    # exact data against the Float64 oracle bit for bit
    ora, ore, orr = oracle_arburg(imp, 5)
    assert np.array_equal(a[:, 0].astype(ora.dtype), ora) and err[0] == R.type(ore)
    # p = n (Burg), p = n - 1 (Levinson), n = 1
    x = _data(T, 9, 1, 2)[:, 0]
    ga, ge, gr = dsp.arburg(x, 9)
    ea, ee, er = exact_arburg(x, 9)
    assert same_bits(ga, ea) and same_bits(ge, ee) and same_bits(gr, er)
    ga, ge = dsp.lpc(x, 8, dsp.LPCLevinson())
    ea, ee = exact_lpc(x, 8, "levinson")
    assert same_bits(ga, ea) and same_bits(ge, ee)
    for p in (0, 1):
        ga, ge, gr = dsp.arburg(x[:1], p)
        ea, ee, er = exact_arburg(x[:1], p)
        assert same_bits(ga, ea) and same_bits(ge, ee) and same_bits(gr, er)


@pytest.fixture
def torch():
    return pytest.importorskip("torch")


_TDT = {np.dtype(np.float32): "float32", np.dtype(np.float64): "float64", np.dtype(np.complex64): "complex64",
        np.dtype(np.complex128): "complex128"}


@pytest.mark.gpu
@pytest.mark.parametrize("T", DTYPES)
def test_guard_cells_streams_and_graphs(T, torch):
    T = np.dtype(T)
    R = _real(T)
    G = 64
    n, ncols, p = 3000, 3, 12
    x = _data(T, n, ncols, 9)
    xt = torch.from_numpy(x.T.copy()).cuda()                       # row c of xt is column c of x
    cases = []
    for name, na, wb in (("burg", p + 1, dsp._lib.lpc_work_bytes(T, n, ncols, p, 0, 2)),
                         ("levinson", p, dsp._lib.lpc_work_bytes(T, n, ncols, p, 1))):
        cases.append((name, na, wb))
    ref = {"burg": dsp.arburg(x, p), "levinson": dsp.lpc(x, p, dsp.LPCLevinson())}
    tdt = getattr(torch, _TDT[T])
    rdt = getattr(torch, _TDT[R])
    for name, na, wb in cases:
        a = torch.full((na * ncols + 2 * G,), float("nan"), dtype=tdt, device="cuda")
        err = torch.full((ncols + 2 * G,), float("nan"), dtype=rdt, device="cuda")
        refl = torch.full((p * ncols + 2 * G,), float("nan"), dtype=tdt, device="cuda")
        work = torch.full((wb + 2 * 1024,), 7, dtype=torch.uint8, device="cuda")
        isz, rsz = T.itemsize, R.itemsize

        def call(stream):
            if name == "burg":
                dsp._lib.lpc_burg_async(T, xt.data_ptr(), n, ncols, p, a.data_ptr() + G * isz, err.data_ptr() + G * rsz,
                                        refl.data_ptr() + G * isz, work.data_ptr() + 1024, 2, stream)
            else:
                dsp._lib.lpc_levinson_async(T, xt.data_ptr(), n, ncols, p, a.data_ptr() + G * isz, err.data_ptr() + G * rsz,
                                            refl.data_ptr() + G * isz, work.data_ptr() + 1024, stream)

        def check():
            torch.cuda.synchronize()
            ah, eh = a.cpu().numpy(), err.cpu().numpy()
            assert np.all(np.isnan(ah[:G])) and np.all(np.isnan(ah[-G:])) and np.all(np.isnan(eh[:G])) and np.all(np.isnan(eh[-G:]))
            wh = work.cpu().numpy()
            assert np.all(wh[:1024] == 7) and np.all(wh[-1024:] == 7)
            got = np.asfortranarray(ah[G:-G].reshape(ncols, na).T)
            assert same_bits(got, ref[name][0]) and same_bits(eh[G:-G], ref[name][1])

        torch.cuda.synchronize()
        call(None)
        check()
        st = torch.cuda.Stream()
        a.fill_(float("nan"))
        with torch.cuda.stream(st):
            torch.cuda._sleep(20_000_000)
            call(st.cuda_stream)
        st.synchronize()
        check()
        g = torch.cuda.CUDAGraph()
        cs = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=cs):
            call(cs.cuda_stream)
        a.fill_(float("nan"))
        err[G:-G].fill_(float("nan"))
        g.replay()
        check()


@pytest.mark.gpu
def test_a_call_past_element_2_31(torch):
    n, p = 4096, 4
    ncols = (1 << 31) // n + 2
    x = torch.randn(n * ncols, dtype=torch.float32, device="cuda")
    a = torch.empty((p + 1) * ncols, dtype=torch.float32, device="cuda")
    err = torch.empty(ncols, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    dsp._lib.lpc_burg_async(np.float32, x.data_ptr(), n, ncols, p, a.data_ptr(), err.data_ptr(), None, None, 0)
    torch.cuda.synchronize()
    ah, eh = a.cpu().numpy().reshape(ncols, p + 1), err.cpu().numpy()
    for c in (0, ncols // 2, ncols - 2, ncols - 1):
        col = x[c * n:(c + 1) * n].cpu().numpy()
        av, ev, _ = dsp.arburg(col, p)
        assert same_bits(ah[c], av) and same_bits(eh[c], ev), c
    del x
    torch.cuda.empty_cache()
