"""Stateful FIR filtering: PolynomialRatio, DF2TFilter and the deprecated filt(b, a, x, si) forms (src/Filters/filt.jl:100-224,
src/deprecated.jl), on the STATE instances of the tiled FIR kernel.

The property checked throughout: in transposed direct form the FIR state is the partial fused multiply-add chain of the
next nb - 1 outputs, so a signal filtered chunk by chunk is bit-identical to the signal filtered in one call (and, from a
zero state, to the stateless filt(b, 1, x)).  The DF2T oracle below restates the reference loop with the state carried in
and out; it lives with the tests that use it."""
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from conftest import ROOT, relerr

import dspb200 as dsp
from dspb200 import _lib
from dspb200.device import DeviceArray
from oracle import dspbase as od

DTYPES = [np.float32, np.float64, np.complex64, np.complex128]


# =============================================================================== oracle (test infrastructure)

def _fma_exact(a, b, c, T):
    """Correctly rounded fused multiply-add in the real dtype T (exact rational arithmetic, one rounding)."""
    if np.dtype(T) == np.float32:
        return od.fma_f32(a, b, c)[()]
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        return np.float64(a) * np.float64(b) + np.float64(c)
    return np.float64(float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))))


def _muladd(x, b, acc, T):
    """muladd(x, b, acc) in eltype T; complex: Base.muladd(z, w, x) of base/complex.jl."""
    T = np.dtype(T)
    if T.kind != "c":
        return _fma_exact(x, b, acc, T)
    R = np.float32 if T == np.complex64 else np.float64
    re = _fma_exact(x.real, b.real, -_fma_exact(x.imag, b.imag, -acc.real, R), R)
    im = _fma_exact(x.real, b.imag, _fma_exact(x.imag, b.real, acc.imag, R), R)
    return T.type(complex(re, im))


def df2t_fir_literal(b, x, si):
    """The reference's _filt_fir! loop (src/dspbase.jl:95-105) on one column with the state carried in and out, every
    muladd a correctly rounded fma in the dtype of the state.  Returns (y, final state).  The newest tap's term is
    muladd(x, b[nb], 0): the reference's product b[nb] * x for real eltypes (up to the sign of a zero)."""
    si = np.array(si, copy=True)
    T = si.dtype
    b = np.asarray(b).astype(T)
    x = np.asarray(x).astype(T)
    ns = b.size - 1
    y = np.empty(x.size, dtype=T)
    zero = T.type(0)
    for i, xi in enumerate(x):
        if ns == 0:
            y[i] = _muladd(xi, b[0], zero, T)
            continue
        y[i] = _muladd(xi, b[0], si[0], T)
        for j in range(ns - 1):
            si[j] = _muladd(xi, b[j + 1], si[j + 1], T)
        si[ns - 1] = _muladd(xi, b[ns], zero, T)
    return y, si


def df2t_fir_f32(b, x, si):
    """Vectorised Float32-faithful form of the same loop for a (nx, ncols) signal and an (nb-1, ncols) state: output i of
    the call is the chain seeded with si[i] (zero for i >= nb-1) over the taps oldest first, samples outside the call's
    [0, nx) being zero; outputs nx .. nx+nb-2 are the final state.  Every step is one correctly rounded fma."""
    b = np.asarray(b, dtype=np.float32)
    x = np.asarray(x, dtype=np.float32).reshape(np.shape(x)[0], -1)
    nx, ncols = x.shape
    ns = b.size - 1
    si = np.asarray(si, dtype=np.float32).reshape(ns, ncols)
    n = nx + ns
    acc = np.zeros((n, ncols), dtype=np.float32)
    acc[:ns] = si
    xp = np.concatenate([np.zeros((ns, ncols), np.float32), x, np.zeros((ns, ncols), np.float32)])
    for k in range(ns, -1, -1):                      # tap k touches sample i - k
        acc = od.fma_f32(xp[ns - k: ns - k + n], b[k], acc)
    return acc[:nx], acc[nx:]


# =============================================================================== CPU: oracle

def test_oracle_reference_cases():
    # test/filt.jl:54-55: a numerator with leading zeros keeps them (coef_z reads from z^0)
    imp = np.r_[1.0, np.zeros(9)]
    y, _ = df2t_fir_literal([0, 0, 1, 0.8], imp, np.zeros(3))
    assert np.array_equal(y, np.r_[0, 0, 1, 0.8, np.zeros(6)])
    assert np.array_equal(od.filt(np.array([0, 0, 1, 0.8]), np.array([1.0]), imp), y)
    # :59: more taps than SMALL_FILT_CUTOFF
    b = np.random.default_rng(59).random(dsp.SMALL_FILT_CUTOFF + 1)
    y, s = df2t_fir_literal(b, np.ones(10), np.zeros(b.size - 1))
    assert np.array_equal(y, od.filt_fir_literal(b, np.ones(10))) and s.size == b.size - 1
    # :88-92 multi-column (D = 1..4): every column from a zero state (what the deprecated si forms of :85-86 pass), and the
    # state each column carries on; the deprecated forms themselves are tested with the host front end below and on the GPU
    b = np.array([0.1, 0.1])
    y_ref, _ = df2t_fir_literal(b, np.ones(10), np.zeros(1))
    for D in range(1, 5):
        sz = (10,) + tuple(range(2, D + 2))
        x = np.ones(sz).reshape(10, -1)
        for c in range(x.shape[1]):
            y, s = df2t_fir_literal(b, x[:, c], np.zeros(1))
            assert np.array_equal(y, y_ref) and s[0] == np.float64(0.1)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("nb", [2, 3, 9, 17])
def test_oracle_chunked_equals_one_shot(dt, nb):
    rng = np.random.default_rng(nb)
    def r(*s):
        v = rng.standard_normal(s)
        return (v + 1j * rng.standard_normal(s) if np.dtype(dt).kind == "c" else v).astype(dt)
    b, x, si = r(nb), r(40), r(nb - 1)
    y1, s1 = df2t_fir_literal(b, x, si)
    pieces, s = [], si
    for lo, hi in [(0, 0), (0, 1), (1, nb - 1), (nb - 1, nb), (nb, 2 * nb), (2 * nb, 40)]:
        y, s = df2t_fir_literal(b, x[lo:hi], s)
        pieces.append(y)
    assert np.array_equal(np.concatenate(pieces), y1) and np.array_equal(s, s1)
    if np.dtype(dt) == np.float32:                   # the vectorised form is the same chain
        yv, sv = df2t_fir_f32(b, x, si)
        assert np.array_equal(yv[:, 0], y1) and np.array_equal(sv[:, 0], s1)


# =============================================================================== CPU: host emulation of the kernel

def test_host_fir_state_emulation():
    """The STATE body of fir_tile_kernel (fir_tile.cuh) compiled for the host: every "thread" of every CTA, all four element
    types, tap counts around the 8-tap chunk and 512-tap staging-round boundaries, chunk lengths 0, 1, nb-2, nb-1, nb and
    several tiles; outputs and final state bit for bit against the literal DF2T loop, chunked calls against one call."""
    exe = os.path.join(ROOT, "build", "fir_state_host_check")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    src = os.path.join(ROOT, "tests", "host", "fir_state_host_check.cu")
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(src), os.path.getmtime(
            os.path.join(ROOT, "dsp.jl_b200", "csrc", "fir_tile.cuh"))):
        subprocess.run(["g++", "-std=c++17", "-O2", "-march=native", "-x", "c++", "-w", "-I/usr/local/cuda/include", "-o", exe, src],
                       check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-2000:]


# =============================================================================== CPU: host bookkeeping with a stand-in library

class _FakeFirPlan:
    """numpy model of dspb200_fir_exec_state's contract (the vectorised oracle for Float32, the literal loop otherwise)."""
    calls = []

    def __init__(self, b):
        self.b = np.ascontiguousarray(b)
        self.dtype = self.b.dtype

    def exec_state(self, x, nx, ncols, si_in, si_out, out):
        ns = self.b.size - 1
        assert x.dtype == out.dtype == self.dtype and x.flags.f_contiguous and out.flags.f_contiguous
        assert x.shape == out.shape == (nx, ncols) and nx > 0 and ncols > 0
        for s in (si_in, si_out):
            assert s is None if ns == 0 else (s.shape == (ns, ncols) and s.dtype == self.dtype and s.flags.f_contiguous)
        _FakeFirPlan.calls.append((nx, ncols))
        for c in range(ncols):
            y, s = df2t_fir_literal(self.b, x[:, c], np.zeros(ns, self.dtype) if si_in is None else si_in[:, c])
            out[:, c] = y
            if si_out is not None:
                si_out[:, c] = s

    def close(self):
        pass


@pytest.fixture
def fake_lib(monkeypatch):
    monkeypatch.setattr(_lib, "FirPlan", _FakeFirPlan)
    _FakeFirPlan.calls = []
    return _FakeFirPlan


def test_polynomialratio_normalisation_eltype_and_trimming():
    f = dsp.PolynomialRatio([1, 2, 3], [2, 3, 4])                  # src/Filters/coefficients.jl:110-111
    assert np.array_equal(f.coefb, [0.5, 1.0, 1.5]) and np.array_equal(f.coefa, [1.0, 1.5, 2.0])
    assert f.coefb.dtype == np.float64                            # typeof(one(Int) / one(Int))
    assert dsp.PolynomialRatio(np.float32([1, 2]), 3).coefb.dtype == np.float32       # Float32 / Int -> Float32
    assert dsp.PolynomialRatio([1, 2], np.float32(3)).coefb.dtype == np.float32
    assert dsp.PolynomialRatio(np.float32([1]), [2.0]).coefb.dtype == np.float64
    assert dsp.PolynomialRatio(np.complex64([1j]), [1]).coefb.dtype == np.complex64
    assert np.array_equal(dsp.PolynomialRatio([0, 0, 1, 0.8], [1]).coefb, [0, 0, 1, 0.8])    # test/filt.jl:54
    assert np.array_equal(dsp.PolynomialRatio([1, 2, 0, 0], [1, 0.5, 0]).coefb, [1, 2])      # zeros of the oldest powers go
    assert np.array_equal(dsp.PolynomialRatio([1, 2, 0, 0], [1, 0.5, 0]).coefa, [1, 0.5])
    assert np.array_equal(dsp.PolynomialRatio([0, 0], [1]).coefb, [0.0])
    assert np.array_equal(dsp.PolynomialRatio(3.7, 4.2).coefb, [3.7 / 4.2])
    assert dsp.coefb(f) is f.coefb and dsp.coefa(f) is f.coefa
    with pytest.raises(dsp.ArgumentError):
        dsp.PolynomialRatio([1], [0, 1])
    with pytest.raises(dsp.ArgumentError):
        dsp.PolynomialRatio([1], [])


def test_df2t_constructors_and_state_shapes():
    pr = dsp.PolynomialRatio([1.0, 2, 3, 4], [1])
    assert dsp.DF2TFilter(pr).state.shape == (3,) and dsp.DF2TFilter(pr).state.dtype == np.float64
    assert dsp.DF2TFilter(pr, (5,)).state.shape == (3, 5)
    assert dsp.DF2TFilter(pr, (2, 3)).state.shape == (3, 2, 3)
    f = dsp.DF2TFilter(pr, np.complex64, (4,))
    assert f.state.shape == (3, 4) and f.state.dtype == np.complex128           # promote_type(T, V)
    assert dsp.DF2TFilter(dsp.PolynomialRatio(np.float32([1, 2]), 1), np.float32).state.dtype == np.float32
    si = np.arange(6.0).reshape(3, 2)
    assert dsp.DF2TFilter(pr, si).state is si                                   # the reference keeps the caller's array
    assert dsp.DF2TFilter(dsp.PolynomialRatio([3.7], [4.2])).state.shape == (0,)
    with pytest.raises(dsp.ArgumentError, match="length of state vector must match filter order"):
        dsp.DF2TFilter(pr, np.zeros(2))
    with pytest.raises(dsp.ArgumentError, match="length of state vector must match filter order"):
        dsp.DF2TFilter(pr, np.zeros((4, 2)))
    for bad in (((5,), (2,)), ((5,), np.float32), (np.float32, 5), (np.float32, (5,), (2,)), (si, (2,))):
        with pytest.raises(TypeError):                                          # a MethodError in the reference
            dsp.DF2TFilter(pr, *bad)
    with pytest.raises(NotImplementedError):
        dsp.DF2TFilter(dsp.PolynomialRatio([1], [1, -0.5]))                    # IIR stays out of scope
    with pytest.raises(NotImplementedError):
        dsp.DF2TFilter(np.ones(3))


def test_df2t_host_filter_carries_state_and_checks_sizes(fake_lib):
    rng = np.random.default_rng(11)
    b = rng.standard_normal(5)
    x = rng.standard_normal((23, 2, 3))
    f = dsp.DF2TFilter(dsp.PolynomialRatio(b, 1), (2, 3))
    st = f.state
    pieces = [dsp.filt(f, x[lo:hi]) for lo, hi in [(0, 3), (3, 3), (3, 4), (4, 23)]]
    assert f.state is st                                                        # updated in place
    y = np.concatenate(pieces)
    for i in range(2):
        for j in range(3):
            want, s = df2t_fir_literal(b, x[:, i, j], np.zeros(4))
            assert np.array_equal(y[:, i, j], want) and np.array_equal(st[:, i, j], s)
    assert fake_lib.calls == [(3, 6), (1, 6), (19, 6)]                          # the empty chunk does no work
    out = np.empty((4, 2, 3))
    assert dsp.filt_(out, f, x[:4]) is out
    with pytest.raises(dsp.ArgumentError, match="out size must match x"):
        dsp.filt_(np.empty((5, 2, 3)), f, x[:4])
    with pytest.raises(dsp.ArgumentError, match="state size must match x"):
        dsp.filt(f, x[:, 0])
    n = len(fake_lib.calls)
    g = dsp.DF2TFilter(dsp.PolynomialRatio([3.7], [4.2]))                       # nb == 1: no state, x * b[1]
    assert np.array_equal(dsp.filt(g, x[:, 0, 0]), x[:, 0, 0] * (3.7 / 4.2)) and len(fake_lib.calls) == n + 1
    # filt(f::PolynomialRatio, x) is filt(coefb, coefa, x)
    assert np.array_equal(dsp.filt(dsp.PolynomialRatio(b, 2.0), np.zeros(0)), np.zeros(0))
    # in place, as filt!(out, f, x) allows: the host form stages x, so out may be x
    h1, h2 = dsp.DF2TFilter(dsp.PolynomialRatio(b, 1), (2, 3)), dsp.DF2TFilter(dsp.PolynomialRatio(b, 1), (2, 3))
    xi = np.asfortranarray(x.copy())
    want = np.concatenate([dsp.filt(h1, x[:9]), dsp.filt(h1, x[9:])])
    assert dsp.filt_(xi[:9], h2, xi[:9]) is not None and dsp.filt_(xi[9:], h2, xi[9:]) is not None
    assert np.array_equal(xi, want) and np.array_equal(h1.state, h2.state)
    # a complex filter output does not fit a real `out` (InexactError in the reference), before any work
    c = dsp.DF2TFilter(dsp.PolynomialRatio(b, 1), np.complex128, (2, 3))
    n = len(fake_lib.calls)
    with pytest.raises(dsp.InexactError):
        dsp.filt_(np.empty((4, 2, 3)), c, x[:4])
    assert len(fake_lib.calls) == n and not np.any(c.state)


def test_df2t_promotion_and_rejection_table(fake_lib):
    pr64 = dsp.PolynomialRatio([1, 2, 3], [1])                    # Float64 coefficients
    pr32 = dsp.PolynomialRatio(np.float32([1, 2, 3]), np.float32(1))
    x = np.arange(6)
    accepted = [(pr64, None, np.float64, np.float64), (pr64, None, np.float32, np.float64), (pr64, None, np.int64, np.float64),
                (pr32, None, np.float32, np.float32), (pr32, None, np.int16, np.float32),
                (pr64, np.complex128, np.complex128, np.complex128), (pr64, np.complex128, np.float64, np.complex128),
                (pr64, np.complex128, np.complex64, np.complex128), (pr32, np.complex64, np.complex64, np.complex64)]
    for coef, V, X, out in accepted:
        f = dsp.DF2TFilter(coef) if V is None else dsp.DF2TFilter(coef, V)
        y = dsp.filt(f, x.astype(X))
        assert y.dtype == out and f.state.dtype == out, (coef.dtype, V, X)
    rejected = [(pr32, None, np.float64, dsp.ArgumentError),        # the reference rounds the state to Float32 per sample
                (pr32, np.float64, np.float32, dsp.ArgumentError),  # the newest product is formed in Float32
                (pr64, None, np.complex128, dsp.InexactError),
                (pr32, None, np.complex64, dsp.InexactError)]
    for coef, V, X, err in rejected:
        f = dsp.DF2TFilter(coef) if V is None else dsp.DF2TFilter(coef, V)
        before = f.state.copy()
        with pytest.raises(err):
            dsp.filt(f, x.astype(X))
        assert np.array_equal(f.state, before)
    f = dsp.DF2TFilter(pr64, np.zeros(2, dtype=np.float32))            # explicit Float32 state with Float64 taps
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(f, x.astype(np.float32))
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(dsp.DF2TFilter(pr64, np.zeros(2, dtype=np.int64)), x)
    assert fake_lib.calls == [(6, 1)] * len(accepted)


def test_deprecated_si_forms_copy_and_repeat_the_state(fake_lib):
    rng = np.random.default_rng(5)
    b, x = rng.standard_normal(4), rng.standard_normal((12, 3))
    si = rng.standard_normal(3)
    keep = si.copy()
    y = dsp.filt(b, 1.0, x, si)                                         # vector si repeated over the columns
    assert np.array_equal(si, keep)
    for c in range(3):
        assert np.array_equal(y[:, c], df2t_fir_literal(b, x[:, c], si)[0])
    si2 = rng.standard_normal((3, 3))
    keep2 = si2.copy()
    out = np.empty_like(x)
    assert dsp.filt_(out, b, 2.0, x, si2) is out and np.array_equal(si2, keep2)
    for c in range(3):
        assert np.array_equal(out[:, c], df2t_fir_literal(b / 2.0, x[:, c], si2[:, c])[0])
    pr = dsp.PolynomialRatio(b, 1.0)
    assert np.array_equal(dsp.filt(pr, x[:, 0], si), df2t_fir_literal(b, x[:, 0], si)[0])
    out1 = np.empty(12)
    assert np.array_equal(dsp.filt_(out1, pr, x[:, 0], si), df2t_fir_literal(b, x[:, 0], si)[0]) and np.array_equal(si, keep)
    with pytest.raises(NotImplementedError):
        dsp.filt([1.0], [1.0, -0.8], x, np.zeros(1))


class _AddressOnly(DeviceArray):
    """A DeviceArray view over a dummy address: nothing is allocated, read or launched."""

    def __init__(self, shape, dtype, _base=None, _ptr=1 << 20):
        super().__init__(shape, dtype, _base=_base, _ptr=_ptr)


def test_residency_rules_fail_before_any_work(fake_lib, monkeypatch):
    monkeypatch.setattr(dsp.df2t, "DeviceArray", _AddressOnly)
    pr = dsp.PolynomialRatio([1.0, 2.0, 3.0], [1])
    host = dsp.DF2TFilter(pr)
    dev_x = _AddressOnly((8,), np.float64, _ptr=256)
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(host, dev_x)
    with pytest.raises(dsp.ArgumentError):
        dsp.filt_(dev_x, host, np.zeros(8))
    dev = dsp.DF2TFilter(pr, _AddressOnly((2,), np.float64, _ptr=4096))     # second state buffer at 1 << 20
    assert dev.device and isinstance(dev.state, DeviceArray)
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(dev, np.zeros(8))
    with pytest.raises(dsp.ArgumentError):
        dsp.filt_(np.zeros(8), dev, dev_x)
    with pytest.raises(dsp.ArgumentError):                              # device chunks carry the state's eltype
        dsp.filt(dev, _AddressOnly((8,), np.float32))
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(dev, _AddressOnly((8, 2), np.float64))
    with pytest.raises(dsp.ArgumentError):
        dsp.filt([1.0, 2.0], 1.0, np.zeros(8), _AddressOnly((1,), np.float64))
    # no in-place device filtering: out may not overlap x or a state buffer
    for out in (dev_x, _AddressOnly((8,), np.float64, _ptr=256 + 24), _AddressOnly((8,), np.float64, _ptr=256 - 40),
                _AddressOnly((8,), np.float64, _ptr=4096 + 8), _AddressOnly((8,), np.float64)):
        with pytest.raises(dsp.ArgumentError, match="in place"):
            dsp.filt_(out, dev, dev_x)
    assert fake_lib.calls == []


# =============================================================================== GPU

def _rand(rng, shape, dt):
    v = rng.standard_normal(shape)
    if np.dtype(dt).kind == "c":
        v = v + 1j * rng.standard_normal(shape)
    return v.astype(dt)


def _chunks(n, nb, rng, rest_in_one=False):
    """Irregular chunk lengths covering n samples, including 0, 1, nb-2, nb-1, nb (then the rest in one chunk, or in
    random chunks)."""
    want = [0, 1, max(nb - 2, 0), nb - 1, nb, 0, 3]
    out, pos = [], 0
    for c in want:
        c = min(c, n - pos)
        out.append(c)
        pos += c
    while pos < n:
        c = n - pos if rest_in_one else min(int(rng.integers(1, 3000)), n - pos)
        out.append(c)
        pos += c
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("nb", [1, 2, 9, 66, 67, 257, 1030])
def test_chunked_equals_one_shot_and_stateless(dt, nb):
    rng = np.random.default_rng(nb * 7 + np.dtype(dt).itemsize)
    b = _rand(rng, nb, dt)
    # a few columns in random chunks (128-thread instances); 200 columns whose last chunk fills the GPU (256-thread)
    for ncols, n, big in ((3, 9000, False), (200, 14000, True)):
        x = _rand(rng, (n, ncols), dt)
        f = dsp.DF2TFilter(dsp.PolynomialRatio(b, np.ones(1, dt)), np.dtype(dt), (ncols,))
        pieces, pos = [], 0
        for c in _chunks(n, nb, rng, big):
            pieces.append(dsp.filt(f, x[pos:pos + c]))
            pos += c
        y = np.concatenate(pieces)
        stateless = dsp.filt(b, np.ones(1, dt), x)
        assert y.dtype == np.dtype(dt) and np.array_equal(y, stateless)
        g = dsp.DF2TFilter(dsp.PolynomialRatio(b, np.ones(1, dt)), np.dtype(dt), (ncols,))
        assert np.array_equal(dsp.filt(g, x), y) and np.array_equal(g.state, f.state)
        # the final state is the tail of the stateless filter over the zero-extended signal (the same chains)
        ext = dsp.filt(b, np.ones(1, dt), np.concatenate([x, np.zeros((nb - 1, ncols), dt)]))
        assert np.array_equal(f.state, ext[n:])
        if np.dtype(dt) == np.float32 and nb > 1 and not big:
            _, s_or = df2t_fir_f32(b, x, np.zeros((nb - 1, ncols), np.float32))
            assert np.array_equal(f.state, s_or)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("nb", [2, 19, 66, 67, 257, 1500])
def test_random_initial_state_against_the_oracle(dt, nb):
    rng = np.random.default_rng(nb + 100)
    b, x, si = _rand(rng, nb, dt), _rand(rng, (5000, 2), dt), _rand(rng, (nb - 1, 2), dt)
    f = dsp.DF2TFilter(dsp.PolynomialRatio(b, np.ones(1, dt)), si.copy())
    y = np.concatenate([dsp.filt(f, x[:1234]), dsp.filt(f, x[1234:])])
    if np.dtype(dt) == np.float32:
        yo, so = df2t_fir_f32(b, x, si)
        assert np.array_equal(y, yo) and np.array_equal(f.state, so)
    # Float64 truth: the same loop in double (complex: double complex) precision
    W = np.complex128 if np.dtype(dt).kind == "c" else np.float64
    xw = np.concatenate([np.zeros((nb - 1, 2)), x.astype(W), np.zeros((nb - 1, 2))])
    acc = np.zeros((5000 + nb - 1, 2), W)
    acc[:nb - 1] = si
    for k in range(nb - 1, -1, -1):
        acc = acc + xw[nb - 1 - k: nb - 1 - k + 5000 + nb - 1] * W(b[k])
    tol = 1e-5 if np.dtype(dt) in (np.float32, np.complex64) else 1e-13
    assert relerr(y, acc[:5000]) < tol and relerr(f.state, acc[5000:]) < tol
    # small case against the literal loop, every fma correctly rounded
    f2 = dsp.DF2TFilter(dsp.PolynomialRatio(b[:9], np.ones(1, dt)), si[:8, 0].copy())
    y2 = np.concatenate([dsp.filt(f2, x[:5, 0]), dsp.filt(f2, x[5:60, 0])])
    yl, sl = df2t_fir_literal(b[:9], x[:60, 0], si[:8, 0])
    assert np.array_equal(y2, yl) and np.array_equal(f2.state, sl)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_integer_valued_data_is_exact(dt):
    rng = np.random.default_rng(3)
    nb, n = 67, 4000
    bi, xi, si = rng.integers(-4, 5, nb), rng.integers(-8, 9, (n, 3)), rng.integers(-50, 51, (nb - 1, 3))
    bi[-1] = 3                                     # a zero oldest tap would shorten the filter (coef_z trimming)
    full = np.zeros((n + nb - 1, 3), dtype=np.int64)
    full[:nb - 1] = si
    for k in range(nb):
        full[k:k + n] += bi[k] * xi
    f = dsp.DF2TFilter(dsp.PolynomialRatio(bi.astype(dt), np.ones(1, dt)), si.astype(dt))
    y = np.concatenate([dsp.filt(f, xi[:100].astype(dt)), dsp.filt(f, xi[100:].astype(dt))])
    assert np.array_equal(y, full[:n].astype(dt)) and np.array_equal(f.state, full[n:].astype(dt))


@pytest.mark.gpu
def test_reference_cases_on_the_device():
    imp = np.r_[1.0, np.zeros(9)]
    assert np.array_equal(dsp.filt(dsp.DF2TFilter(dsp.PolynomialRatio([0, 0, 1, 0.8], [1])), imp), np.r_[0, 0, 1, 0.8, np.zeros(6)])
    assert np.array_equal(dsp.filt([0, 0, 1, 0.8], [1], imp), np.r_[0, 0, 1, 0.8, np.zeros(6)])       # test/filt.jl:54-55
    x = np.random.default_rng(0).standard_normal(100)
    assert np.array_equal(dsp.filt(dsp.DF2TFilter(dsp.PolynomialRatio([3.7], [4.2])), x), x * (3.7 / 4.2))   # :51
    dsp.filt(dsp.DF2TFilter(dsp.PolynomialRatio(np.random.default_rng(1).random(dsp.SMALL_FILT_CUTOFF + 1), [1])), np.ones(10))
    b, a = [0.1, 0.1], [1.0]
    for D in range(1, 5):                                                  # :88-93 and the DF2TFilter block :95-104 (FIR)
        sz = (10,) + tuple(range(2, D + 2))
        y_ref = dsp.filt(b, a, np.ones(10))
        y2_ref = dsp.filt(b, a, np.ones(20))
        xs = np.ones(sz)
        cols = lambda y: y.reshape(10, -1).T
        assert all(np.array_equal(c, y_ref) for c in cols(dsp.filt(b, a, xs)))
        assert all(np.array_equal(c, y_ref) for c in cols(dsp.filt(dsp.PolynomialRatio(b, a), xs)))
        assert all(np.array_equal(c, y_ref) for c in cols(dsp.filt(b, a, xs, np.zeros((1,) + sz[1:]))))
        assert all(np.array_equal(c, y_ref) for c in cols(dsp.filt(dsp.PolynomialRatio(b, a), xs, np.zeros((1,) + sz[1:]))))
        H = dsp.DF2TFilter(dsp.PolynomialRatio(b, a), sz[1:])
        assert all(np.array_equal(c, y2_ref[:10]) for c in cols(dsp.filt(H, xs)))
        assert all(np.array_equal(c, y2_ref[10:]) for c in cols(dsp.filt(H, xs)))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_device_filter_matches_host_filter_one_launch_per_chunk(dt):
    rng = np.random.default_rng(21)
    nb, n, ncols = 257, 20000, 4
    b, x, si = _rand(rng, nb, dt), _rand(rng, (n, ncols), dt), _rand(rng, (nb - 1, ncols), dt)
    pr = dsp.PolynomialRatio(b, np.ones(1, dt))
    host = dsp.DF2TFilter(pr, si.copy())
    dev = dsp.DF2TFilter(pr, si.copy(), device=True)
    dx = dsp.to_device(x)
    bounds = [0, 0, 1, 255, 256, 257, 4096, 4096, 20000]
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        yh = dsp.filt(host, x[lo:hi])
        chunk = DeviceArray((hi - lo, ncols), dt)
        chunk.copy_from_host(x[lo:hi])
        before = dsp.launch_count()
        yd = dsp.filt(dev, chunk)
        assert dsp.launch_count() - before == (1 if hi > lo else 0)
        assert isinstance(yd, DeviceArray) and np.array_equal(yd.to_host(), yh)
        assert np.array_equal(dev.state.to_host(), host.state)
    out = DeviceArray((n, ncols), dt)
    g = dsp.DF2TFilter(pr, dsp.to_device(si), device=False)               # a DeviceArray state makes the filter device-resident
    assert dsp.filt_(out, g, dx) is out
    assert np.array_equal(out.to_host(), dsp.filt(dsp.DF2TFilter(pr, si.copy()), x))
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(g, x)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_stateless_filt_of_a_device_array_equals_the_host_call(dt):
    rng = np.random.default_rng(8)
    b, x = _rand(rng, 67, dt), _rand(rng, (3000, 3), dt)
    y = dsp.filt(b, np.ones(1, dt), dsp.to_device(x))
    assert isinstance(y, DeviceArray) and np.array_equal(y.to_host(), dsp.filt(b, np.ones(1, dt), x))
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(b.astype(np.complex128), 1, dsp.to_device(x.astype(np.complex64)))


@pytest.mark.gpu
def test_argument_errors_fail_before_any_launch():
    pr = dsp.PolynomialRatio(np.ones(9), [1])
    f = dsp.DF2TFilter(pr, (2,))
    dev = dsp.DF2TFilter(pr, (2,), device=True)
    g = dsp.DF2TFilter(pr, (1,), device=True)
    dx = dsp.to_device(np.zeros((16, 2)))
    before = dsp.launch_count()
    for call in (lambda: dsp.filt(f, np.zeros((16, 3))), lambda: dsp.filt(f, np.zeros(16, np.complex128)),
                 lambda: dsp.filt(f, dx), lambda: dsp.filt(dev, np.zeros((16, 2))),
                 lambda: dsp.filt(dev, dsp.to_device(np.zeros((16, 2), np.float32))),
                 lambda: dsp.filt_(DeviceArray((15, 2), np.float64), dev, dx),
                 lambda: dsp.filt_(dx, dev, dx),                                  # in place on the device
                 lambda: dsp.filt_(g.state, g, DeviceArray((8, 1), np.float64)),    # out is the filter's own state
                 lambda: dsp.DF2TFilter(pr, np.zeros(3)), lambda: dsp.filt(np.ones(3), [1.0, 0.5], dx)):
        with pytest.raises((dsp.ArgumentError, dsp.InexactError, NotImplementedError)):
            call()
    assert dsp.launch_count() == before
    # the C ABI refuses overlapping device state buffers
    plan = _lib.FirPlan(np.ones(9))
    s = DeviceArray((8, 2), np.float64)
    s2, o = DeviceArray((8, 2), np.float64), DeviceArray((16, 2), np.float64)
    with pytest.raises(_lib.DSPB200Error):
        plan.exec_state_dev(dx.ptr, 16, 2, s.ptr, s.ptr + 8, o.ptr, 0)
    for x_ptr, out_ptr, si_out_ptr in ((dx.ptr, dx.ptr, s2.ptr), (dx.ptr, dx.ptr + 64, s2.ptr),
                                       (dx.ptr, o.ptr, dx.ptr + 8), (dx.ptr, o.ptr, o.ptr)):
        with pytest.raises(_lib.DSPB200Error, match="overlap"):            # x / out / state ranges may not overlap
            plan.exec_state_dev(x_ptr, 16, 2, s.ptr, si_out_ptr, out_ptr, 0)
    with pytest.raises(_lib.DSPB200Error, match="overlap"):
        plan.exec_state_dev(dx.ptr, 16, 2, o.ptr + 8, s2.ptr, o.ptr, 0)    # si_in inside out
    assert dsp.launch_count() == before
    plan.exec_state_dev(dx.ptr, 16, 2, s.ptr, s2.ptr, o.ptr, 0)              # disjoint buffers: one launch
    assert dsp.launch_count() == before + 1
    plan.close()
    # the host forms stage x, so filtering in place there is the same as filtering into a new array
    rng = np.random.default_rng(4)
    x, si = rng.standard_normal((300, 2)), rng.standard_normal((8, 2))
    want = dsp.filt(dsp.DF2TFilter(pr, si.copy()), x)
    xi = np.asfortranarray(x.copy())
    dsp.filt_(xi, dsp.DF2TFilter(pr, si.copy()), xi)
    assert np.array_equal(xi, want)
    pl = _lib.FirPlan(np.ones(9))
    xc, sc = np.asfortranarray(x.copy()), np.asfortranarray(si.copy())
    pl.exec_state(xc, 300, 2, sc, sc, xc)                                        # x == out and si_in == si_out
    assert np.array_equal(xc, want)
    pl.close()
