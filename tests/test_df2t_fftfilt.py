"""fftfilt(f::DF2TFilter, x): a DF2TFilter's chunked stream through the stateful overlap-save instances
(csrc/overlap_save.cu, `os_fused_kernel<T, N, CPLX, STATE = true>` and the generic path's `os_scatter_kernel<..., true>`).

For an FIR filter in transposed direct form, one chunk x (nx samples per column) with incoming state si_in (nb - 1 values
per column) gives, with full = conv(b, x) (nx + nb - 1 outputs):

    full'[i] = full[i] + (i < nb - 1 ? si_in[i] : 0),   out = full'[0 : nx],   si_out = full'[nx : nx + nb - 1]

for every nx >= 1, nx < nb - 1 included (there si_out[j] picks up si_in[nx + j]).  This is the state of the time-domain
DF2TFilter, so one filter may go through filt and fftfilt in any order, and the GPU tests compare the two exactly.

Exactness on the GPU.  Samples are integers in [-8, 8], taps nonzero integers in [-4, 4] and the initial state integers in
[-50, 50] (both parts of complex data), so every true output and state entry is an integer, and the time-domain filter
computes it exactly.  Error bound: the overlap-save result of one chunk is off by at most e = 0.003 from the integer
convolution (Float32, N = 16384, up to 16384 taps, outputs up to 1.1e4: tests/test_os_kernel_paths.py); the fold adds two
floats below 2^15 per state entry, which rounds by at most 2^-9 in Float32.  A state entry carried through m consecutive
chunks shorter than nb - 1 collects m + 1 of these errors before it is emitted or consumed.  The chunk splits below have at
most four consecutive short chunks, so every output and state entry is within 5 (e + 2^-9) < 0.026 < 2^-4 of its integer
(Float64: far inside 1e-9), which is the bound checked; rint of each must equal the time-domain value bit for bit.

The CPU tests check the fold against the literal DF2T recurrence, restate the routing to show that the GPU case table
reaches every STATE instance and the generic path, and check the front end's rules with a stand-in library."""
import math

import numpy as np
import pytest

import dspb200 as dsp
from dspb200 import _lib
from dspb200.device import DeviceArray

F32, F64, C64, C128 = (np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))
DTYPES = (F32, F64, C64, C128)
GUARD = 64                # sentinel / NaN cells on each side of a device buffer


def _cplx(dt):
    return np.dtype(dt).kind == "c"


def _f64(dt):
    return np.dtype(dt) in (F64, C128)


# =============================================================================== restated routing (csrc/overlap_save.cu)

def auto_nfft(nv, f64):
    """auto_nfft: the cheapest power of two 1024 .. 16384 (Float64: 8192) that leaves half of each block as new output,
    else the generic path's power of two >= 4 nv (from 4096)."""
    nmax = 8192 if f64 else 16384
    best, best_cost = 0, 0.0
    n = 1024
    while n <= nmax:
        if n - nv + 1 >= n / 2:
            cost = n * (math.log2(n) + 2.0) / (n - nv + 1)
            if best == 0 or cost < best_cost:
                best, best_cost = n, cost
        n <<= 1
    if best:
        return best
    n = 4096
    while n < 4 * nv:
        n <<= 1
    return n


def os_fused_ok(nfft, nv, f64):
    return 32 <= nfft <= (8192 if f64 else 16384) and nfft & (nfft - 1) == 0 and nfft >= nv


STATE_SIZES = {F32: (1024, 2048, 4096, 8192, 16384), F64: (1024, 2048, 4096, 8192)}
# tap counts of the GPU table: each reaches one STATE instance (fused nfft) or the generic path ("generic")
NB_TABLE = {F32: (67, 257, 300, 700, 4097, 8200), F64: (67, 257, 300, 700, 4097, 4100)}
NB_TABLE[C64], NB_TABLE[C128] = NB_TABLE[F32], NB_TABLE[F64]
GPU_CASES = [(dt, nb) for dt in DTYPES for nb in NB_TABLE[dt]]


def _route(dt, nb):
    N = auto_nfft(nb, _f64(dt))
    return N if os_fused_ok(N, nb, _f64(dt)) else "generic"


def _chunks(nb, L, rng):
    """Chunk lengths 1, nb - 1, nb, L - 1, L + 1, 4 L (interior units for every instance) and three random lengths in
    [1, L]."""
    return [1, nb - 1, nb, L - 1, L + 1, 4 * L] + [int(v) for v in rng.integers(1, L + 1, 3)]


def _state_units(N, cplx, nv, nx, with_state_out=True):
    """The fused kernel's units of one stateful column (geometry in os_fused_kernel): for each unit the global outputs of
    its block(s) and whether it is interior."""
    L = N - nv + 1
    span = N if cplx else N + L
    count = nx + (nv - 1 if with_state_out else 0)
    nblk = -(-count // L)
    units = []
    for unit in range(nblk if cplx else (nblk + 1) // 2):
        q = unit if cplx else 2 * unit
        s0 = q * L - (nv - 1)
        interior = s0 >= 0 and nx - s0 >= span and count - s0 >= span
        blocks = [[o for o in range(s0 + nv - 1, s0 + N) if o < count]]
        if not cplx:
            blocks.append([o for o in range(s0 + nv - 1 + L, s0 + N + L) if o < count])
        units.append(dict(interior=interior, blocks=blocks))
    return units


# =============================================================================== CPU: the fold against the recurrence

def df2t_literal(b, x, si):
    """The transposed direct-form loop (src/dspbase.jl:95-105) on one column in Float64, state carried in and out."""
    si = np.array(si, dtype=np.float64, copy=True)
    ns = b.size - 1
    y = np.empty(x.size)
    for i, xi in enumerate(x):
        if ns == 0:
            y[i] = xi * b[0]
            continue
        y[i] = xi * b[0] + si[0]
        for j in range(ns - 1):
            si[j] = xi * b[j + 1] + si[j + 1]
        si[ns - 1] = xi * b[ns]
    return y, si


def fold(b, x, si):
    """One chunk by the fold: conv, the incoming state added to the first nb - 1 outputs, the last nb - 1 split off."""
    ns = b.size - 1
    full = np.convolve(x, b)
    full[:ns] += si
    return full[:x.size], full[x.size:]


@pytest.mark.parametrize("nb", [2, 3, 9, 17])
@pytest.mark.parametrize("ncols", [1, 3])
def test_fold_equals_df2t_recurrence(nb, ncols):
    rng = np.random.default_rng([nb, ncols])
    splits = [1, max(nb - 2, 1), nb - 1, nb, 1, 1] + [int(v) for v in rng.integers(1, 2 * nb + 3, 6)]
    n = sum(splits)
    for integer in (True, False):
        if integer:
            b = rng.integers(-4, 5, nb).astype(float)
            b[b == 0] = 3
            x = rng.integers(-8, 9, (n, ncols)).astype(float)
            si0 = rng.integers(-50, 51, (nb - 1, ncols)).astype(float)
        else:
            b, x, si0 = rng.standard_normal(nb), rng.standard_normal((n, ncols)), rng.standard_normal((nb - 1, ncols))
        for c in range(ncols):
            s_lit, s_fold, pos = si0[:, c].copy(), si0[:, c].copy(), 0
            for m in splits:
                xc = x[pos:pos + m, c]
                pos += m
                y_lit, s_lit = df2t_literal(b, xc, s_lit)
                y_fold, s_fold = fold(b, xc, s_fold)
                if integer:
                    assert np.array_equal(y_lit, y_fold) and np.array_equal(s_lit, s_fold), (nb, m)
                else:
                    assert np.allclose(y_lit, y_fold, rtol=0, atol=1e-12) and np.allclose(s_lit, s_fold, rtol=0, atol=1e-12)
            # the whole chunked stream is one call over the concatenation
            assert pos == n
            y1, s1 = df2t_literal(b, x[:, c], si0[:, c])
            assert np.allclose(s1, s_lit, rtol=0, atol=1e-12)


# =============================================================================== CPU: routing coverage

def test_routing_reaches_every_state_instance_and_the_generic_path():
    assert [auto_nfft(nb, False) for nb in NB_TABLE[F32]] == [1024, 2048, 4096, 8192, 16384, 65536]
    assert [auto_nfft(nb, True) for nb in NB_TABLE[F64]] == [1024, 2048, 4096, 8192, 8192, 32768]
    instances = set()
    for dt in DTYPES:
        base = F64 if _f64(dt) else F32
        routes = {_route(dt, nb) for nb in NB_TABLE[dt]}
        assert routes == set(STATE_SIZES[base]) | {"generic"}, dt
        instances |= {(dt, r) for r in routes if r != "generic"}
        # the fused sizes below 1024 have no STATE instance, and auto_nfft never picks them
        assert min(auto_nfft(nb, _f64(dt)) for nb in range(1, 9000)) == 1024
    assert len(instances) == 18
    # every instance sees, over the chunk splits: units taking incoming state, units emitting outgoing state, one unit
    # doing both (a short chunk), interior units -- and the interior units touch no state entry
    for dt, nb in GPU_CASES:
        N = _route(dt, nb)
        if N == "generic":
            continue
        L = N - nb + 1
        seen = dict(seed=False, tail=False, both=False, interior=False, tail_in_b=False)
        for nx in _chunks(nb, L, np.random.default_rng(0)):
            for u in _state_units(N, _cplx(dt), nb, nx):
                outs = [o for blk in u["blocks"] for o in blk]
                seed, tail = any(o < nb - 1 for o in outs), any(o >= nx for o in outs)
                if u["interior"]:
                    assert not seed and not tail and outs and min(outs) >= nb - 1 and max(outs) < nx
                seen["seed"] |= seed
                seen["tail"] |= tail
                seen["both"] |= seed and tail
                seen["interior"] |= u["interior"]
                seen["tail_in_b"] |= len(u["blocks"]) == 2 and any(o >= nx for o in u["blocks"][1])
        if _cplx(dt):
            seen["tail_in_b"] = True
        assert all(seen.values()), (dt, nb, seen)


# =============================================================================== CPU: front end with a stand-in library

class _FakePlan:
    """numpy model of exec_state / exec_state_dev (the fold); records which plan kind ran."""
    calls = []
    kind = None

    def __init__(self, b, nfft=0):
        self.b = np.ascontiguousarray(b)
        self.dtype = self.b.dtype
        self.nfft = nfft

    def exec_state(self, x, nx, ncols, si_in, si_out, out):
        ns = self.b.size - 1
        assert x.dtype == out.dtype == self.dtype and x.flags.f_contiguous and out.flags.f_contiguous
        assert x.shape == out.shape == (nx, ncols) and nx > 0 and ncols > 0
        _FakePlan.calls.append((self.kind, nx, ncols))
        for c in range(ncols):
            y, s = fold(self.b.astype(np.complex128), x[:, c].astype(np.complex128),
                        np.zeros(ns) if si_in is None else si_in[:, c])
            out[:, c] = y if self.dtype.kind == "c" else y.real
            if si_out is not None:
                si_out[:, c] = s if self.dtype.kind == "c" else s.real

    def exec_state_dev(self, x_ptr, nx, ncols, si_in_ptr, si_out_ptr, out_ptr, stream=0):
        _FakePlan.calls.append((self.kind, "dev", nx, ncols, x_ptr, si_in_ptr, si_out_ptr, out_ptr))

    def close(self):
        pass


class _FakeFir(_FakePlan):
    kind = "fir"


class _FakeOs(_FakePlan):
    kind = "os"

    def __init__(self, b, nfft=0):
        assert nfft == 0                           # the stateful form plans with the library's block transform
        super().__init__(b, nfft)


@pytest.fixture
def fake_lib(monkeypatch):
    monkeypatch.setattr(_lib, "FirPlan", _FakeFir)
    monkeypatch.setattr(_lib, "OsPlan", _FakeOs)
    _FakePlan.calls = []
    return _FakePlan


class _AddressOnly(DeviceArray):
    """A DeviceArray view over a dummy address: nothing is allocated, read or launched."""

    def __init__(self, shape, dtype, _base=None, _ptr=1 << 20):
        super().__init__(shape, dtype, _base=_base, _ptr=_ptr)


def test_filt_runs_the_fir_plan_and_fftfilt_the_overlap_save_plan(fake_lib):
    rng = np.random.default_rng(2)
    b = rng.integers(-4, 5, 6).astype(float)
    b[-1] = 2
    x = rng.integers(-8, 9, (40, 2, 3)).astype(float)
    pr = dsp.PolynomialRatio(b, 1)
    f, g = dsp.DF2TFilter(pr, (2, 3)), dsp.DF2TFilter(pr, (2, 3))
    y_fft = np.concatenate([dsp.fftfilt(f, x[:3]), dsp.fftfilt(f, x[3:3]), dsp.filters.fftfilt(f, x[3:25])])
    out = np.empty((15, 2, 3))
    assert dsp.fftfilt_(out, f, x[25:]) is out
    y_fft = np.concatenate([y_fft, out])
    assert [c[0] for c in fake_lib.calls] == ["os"] * 3 and [c[1] for c in fake_lib.calls] == [3, 22, 15]
    fake_lib.calls = []
    y_td = np.concatenate([dsp.filt(g, x[:10]), dsp.filt(g, x[10:])])
    assert [c[0] for c in fake_lib.calls] == ["fir", "fir"]
    assert np.array_equal(y_fft, y_td) and np.array_equal(f.state, g.state)      # one state, two algorithms
    # filt and fftfilt alternate on one filter
    h = dsp.DF2TFilter(pr, (2, 3))
    y_mix = np.concatenate([dsp.filt(h, x[:7]), dsp.fftfilt(h, x[7:8]), dsp.filt(h, x[8:30]), dsp.fftfilt(h, x[30:])])
    assert np.array_equal(y_mix, y_td) and np.array_equal(h.state, g.state)
    # in place on the host (x is staged)
    k = dsp.DF2TFilter(pr, (2, 3))
    xi = np.asfortranarray(x.copy())
    dsp.fftfilt_(xi, k, xi)
    assert np.array_equal(xi, y_td)
    # the stateless forms are unchanged: fftfilt(b, x) takes real data and an nfft; the stateful form takes no nfft
    with pytest.raises(dsp.ArgumentError):
        dsp.fftfilt(f, x, 1024)
    with pytest.raises(dsp.ArgumentError):
        dsp.fftfilt_(out, f, x[:15], 1024)
    with pytest.raises(TypeError):
        dsp.fftfilt(b.astype(complex), x[:, 0, 0])


def test_eltype_table_shapes_and_residency_fail_before_any_work(fake_lib, monkeypatch):
    pr64 = dsp.PolynomialRatio([1, 2, 3], [1])
    pr32 = dsp.PolynomialRatio(np.float32([1, 2, 3]), np.float32(1))
    x = np.arange(6)
    accepted = [(pr64, None, np.float64, np.float64), (pr64, None, np.float32, np.float64), (pr64, None, np.int64, np.float64),
                (pr32, None, np.float32, np.float32), (pr64, np.complex128, np.float64, np.complex128),
                (pr64, np.complex128, np.complex128, np.complex128), (pr32, np.complex64, np.complex64, np.complex64)]
    for coef, V, X, out in accepted:
        f = dsp.DF2TFilter(coef) if V is None else dsp.DF2TFilter(coef, V)
        y = dsp.fftfilt(f, x.astype(X))
        assert y.dtype == out and f.state.dtype == out and f._os.dtype == out, (coef.dtype, V, X)
    rejected = [(pr32, None, np.float64, dsp.ArgumentError), (pr32, np.float64, np.float32, dsp.ArgumentError),
                (pr64, None, np.complex128, dsp.InexactError), (pr32, None, np.complex64, dsp.InexactError)]
    for coef, V, X, err in rejected:
        f = dsp.DF2TFilter(coef) if V is None else dsp.DF2TFilter(coef, V)
        with pytest.raises(err):
            dsp.fftfilt(f, x.astype(X))
    assert fake_lib.calls == [("os", 6, 1)] * len(accepted)
    f = dsp.DF2TFilter(pr64, (2,))
    with pytest.raises(dsp.ArgumentError, match="state size must match x"):
        dsp.fftfilt(f, np.zeros(8))
    with pytest.raises(dsp.ArgumentError, match="out size must match x"):
        dsp.fftfilt_(np.empty((7, 2)), f, np.zeros((8, 2)))
    c = dsp.DF2TFilter(pr64, np.complex128, (2,))
    with pytest.raises(dsp.InexactError):
        dsp.fftfilt_(np.empty((8, 2)), c, np.zeros((8, 2)))
    # residency: a host filter takes host arrays, a device filter DeviceArrays of the state's eltype
    monkeypatch.setattr(dsp.df2t, "DeviceArray", _AddressOnly)
    dev_x = _AddressOnly((8,), np.float64, _ptr=256)
    with pytest.raises(dsp.ArgumentError):
        dsp.fftfilt(dsp.DF2TFilter(pr64), dev_x)
    dev = dsp.DF2TFilter(pr64, _AddressOnly((2,), np.float64, _ptr=4096))     # second state buffer at 1 << 20
    with pytest.raises(dsp.ArgumentError):
        dsp.fftfilt(dev, np.zeros(8))
    with pytest.raises(dsp.ArgumentError):
        dsp.fftfilt_(np.zeros(8), dev, dev_x)
    with pytest.raises(dsp.ArgumentError):
        dsp.fftfilt(dev, _AddressOnly((8,), np.float32))
    with pytest.raises(dsp.ArgumentError):
        dsp.fftfilt(dev, _AddressOnly((8, 2), np.float64))
    # no in-place device filtering: out may not overlap x or a state buffer
    for out in (dev_x, _AddressOnly((8,), np.float64, _ptr=256 + 24), _AddressOnly((8,), np.float64, _ptr=256 - 40),
                _AddressOnly((8,), np.float64, _ptr=4096 + 8), _AddressOnly((8,), np.float64)):
        with pytest.raises(dsp.ArgumentError, match="in place"):
            dsp.fftfilt_(out, dev, dev_x)
    assert fake_lib.calls == [("os", 6, 1)] * len(accepted)
    # a device chunk goes to exec_state_dev with the two state buffers, which then swap
    out = _AddressOnly((8,), np.float64, _ptr=8192)
    dsp.fftfilt_(out, dev, dev_x)
    assert fake_lib.calls[-1] == ("os", "dev", 8, 1, 256, 4096, 1 << 20, 8192) and dev.state.ptr == 1 << 20
    dsp.filt_(out, dev, dev_x)
    assert fake_lib.calls[-1] == ("fir", "dev", 8, 1, 256, 1 << 20, 4096, 8192) and dev.state.ptr == 4096


# =============================================================================== GPU helpers

def _ints(rng, shape, dt, lo, hi):
    v = rng.integers(lo, hi + 1, shape).astype(np.float64)
    if _cplx(dt):
        v = v + 1j * rng.integers(lo, hi + 1, shape)
    return v.astype(dt)


def _taps(rng, nb, dt):
    b = _ints(rng, nb, dt, -4, 4)
    re = b.real.copy()
    re[re == 0] = 3                              # nonzero taps: a stray sample always shows, and coef_z trims nothing
    return (re + 1j * b.imag).astype(dt) if _cplx(dt) else re.astype(dt)


def _sentinels(rng, n, dt):
    s = rng.choice(np.array([-1000.0, 1000.0]), n)
    if _cplx(dt):
        s = s + 1j * rng.choice(np.array([-1000.0, 1000.0]), n)
    return s.astype(dt)


class Guarded:
    """A device buffer of GUARD cells, n data cells and GUARD cells: sentinels (input) or NaN (output) outside the data."""

    def __init__(self, dt, n, rng=None, data=None):
        from dspb200 import device
        self.dt, self.n = np.dtype(dt), n
        host = np.full(n + 2 * GUARD, np.nan, dtype=dt) if rng is None else _sentinels(rng, n + 2 * GUARD, dt)
        if data is not None:
            host[GUARD:GUARD + n] = np.asarray(data).ravel(order="F")
        self.host = host
        self.buf = device.to_device(host)
        self.ptr = self.buf.ptr + GUARD * self.dt.itemsize

    def data(self, shape):
        h = self.buf.to_host()
        outside = np.concatenate([h[:GUARD], h[GUARD + self.n:]])
        want = np.concatenate([self.host[:GUARD], self.host[GUARD + self.n:]])
        assert np.array_equal(outside, want, equal_nan=True), "a cell outside the buffer's range changed"
        return h[GUARD:GUARD + self.n].reshape(shape, order="F")


def _tol(dt):
    return 1e-9 if _f64(dt) else 2.0 ** -4


def _direct(pr, si, chunks_x):
    """The time-domain device DF2TFilter over the same chunks: [(out, state)] after every chunk."""
    f = dsp.DF2TFilter(pr, dsp.to_device(si))
    res = []
    for xc in chunks_x:
        y = DeviceArray(xc.shape, xc.dtype)
        dsp.filt_(y, f, dsp.to_device(xc))
        res.append((y.to_host(), f.state.to_host()))
    return res


# =============================================================================== GPU: exact, per instance

@pytest.mark.gpu
@pytest.mark.parametrize("ncols", [3, 70])
@pytest.mark.parametrize("dt,nb", GPU_CASES, ids=[f"{dt}-{nb}-{_route(dt, nb)}" for dt, nb in GPU_CASES])
def test_every_state_instance_exact_with_guards(dt, nb, ncols):
    from dspb200 import device
    rng = np.random.default_rng([nb, ncols, dt.num])
    b = _taps(rng, nb, dt)
    plan = _lib.OsPlan(b, 0)
    N = _route(dt, nb)
    assert plan.fused == (N != "generic") and (N == "generic" or plan.nfft == N)
    L = plan.nfft - nb + 1
    chunks = _chunks(nb, L, rng)
    n = sum(chunks)
    x = _ints(rng, (n, ncols), dt, -8, 8)
    si = _ints(rng, (nb - 1, ncols), dt, -50, 50)
    xs = np.split(x, np.cumsum(chunks)[:-1])
    want = _direct(dsp.PolynomialRatio(b, np.ones(1, dt)), si, xs)
    state, worst = si, 0.0
    for xc, (y_td, s_td) in zip(xs, want):
        nx = xc.shape[0]
        gx = Guarded(dt, xc.size, rng=rng, data=xc)
        gsi = Guarded(dt, state.size, rng=rng, data=state)
        go, gso = Guarded(dt, xc.size), Guarded(dt, state.size)
        n0 = dsp.launch_count()
        plan.exec_state_dev(gx.ptr, nx, ncols, gsi.ptr, gso.ptr, go.ptr, 0)
        device.sync()
        if plan.fused:
            assert dsp.launch_count() - n0 == 1
        gx.data(xc.shape)
        gsi.data(state.shape)
        y, state = go.data((nx, ncols)), gso.data((nb - 1, ncols))
        assert np.array_equal(np.rint(y), y_td) and np.array_equal(np.rint(state), s_td), (nx, N)
        worst = max(worst, float(np.max(np.abs(y - y_td))), float(np.max(np.abs(state - s_td))))
    print(f"max|y - exact| {dt} nb={nb} nfft={plan.nfft} ncols={ncols}: {worst:.3g}")
    assert worst <= _tol(dt)
    plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_mixing_filt_and_fftfilt_is_exact(dt):
    rng = np.random.default_rng(dt.num)
    nb, ncols = 257, 5
    b, si = _taps(rng, nb, dt), _ints(rng, (nb - 1, ncols), dt, -50, 50)
    pr = dsp.PolynomialRatio(b, np.ones(1, dt))
    chunks = [1, 256, 257, 2000, 3, 5000, 1900, 4000]
    x = _ints(rng, (sum(chunks), ncols), dt, -8, 8)
    xs = np.split(x, np.cumsum(chunks)[:-1])
    want = _direct(pr, si, xs)
    f = dsp.DF2TFilter(pr, dsp.to_device(si))
    for k, (xc, (y_td, s_td)) in enumerate(zip(xs, want)):
        y = DeviceArray(xc.shape, dt)
        (dsp.fftfilt_ if k % 2 else dsp.filt_)(y, f, dsp.to_device(xc))
        y, s = y.to_host(), f.state.to_host()
        assert np.array_equal(np.rint(y), y_td) and np.array_equal(np.rint(s), s_td), k
        assert max(np.max(np.abs(y - y_td)), np.max(np.abs(s - s_td))) <= _tol(dt)
    # host residency: the same alternation through the host forms
    h = dsp.DF2TFilter(pr, si.copy())
    for k, (xc, (y_td, s_td)) in enumerate(zip(xs, want)):
        y = (dsp.fftfilt if k % 2 else dsp.filt)(h, xc)
        assert np.array_equal(np.rint(y), y_td) and np.array_equal(np.rint(h.state), s_td), k


# =============================================================================== GPU: float data

def _truth(b, x, si):
    """Float64 (complex128) stream truth: conv of the whole signal with the initial state folded in."""
    from scipy import signal as ss
    n, ncols = x.shape
    W = np.complex128
    full = ss.oaconvolve(x.astype(W), b.astype(W)[:, None], axes=0)
    full[:b.size - 1] += si
    return full[:n], full[n:]


def _rint(a, dt):
    """An integer-valued Float64 truth rounded and cast to dt."""
    return np.rint(a if _cplx(dt) else a.real).astype(dt)


def _relerr(a, b):
    return float(np.linalg.norm((a.astype(np.complex128) - b).ravel()) / np.linalg.norm(b.ravel()))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("nb", [67, 1030, 4097])
def test_random_data_against_float64(dt, nb):
    rng = np.random.default_rng([nb, dt.num, 7])
    def r(*s):
        v = rng.standard_normal(s)
        return (v + 1j * rng.standard_normal(s) if _cplx(dt) else v).astype(dt)
    b, x, si = r(nb), r(60000, 3), r(nb - 1, 3)
    yt, st = _truth(b, x, si)
    f = dsp.DF2TFilter(dsp.PolynomialRatio(b, np.ones(1, dt)), dsp.to_device(si))
    ys = []
    for lo, hi in ((0, 5), (5, 5 + nb), (5 + nb, 20000), (20000, 60000)):
        ys.append(dsp.fftfilt(f, dsp.to_device(np.asfortranarray(x[lo:hi]))).to_host())
    tol = 1e-12 if _f64(dt) else 2e-6
    y = np.concatenate(ys)
    assert _relerr(y, yt) < tol and _relerr(f.state.to_host(), st) < tol, (_relerr(y, yt), _relerr(f.state.to_host(), st))


@pytest.mark.gpu
def test_headline_filter_long_stream():
    """The 4097-tap ComplexF32 filter over 2^22 samples in 2^18-sample chunks, against Float64."""
    rng = np.random.default_rng(4097)
    n, c, nb = 1 << 22, 1 << 18, 4097
    b = (rng.standard_normal(nb) + 1j * rng.standard_normal(nb)).astype(np.complex64)
    x = (rng.standard_normal((n, 1)) + 1j * rng.standard_normal((n, 1))).astype(np.complex64)
    si = np.zeros((nb - 1, 1), np.complex64)
    yt, st = _truth(b, x, si)
    f = dsp.DF2TFilter(dsp.PolynomialRatio(b, np.ones(1, np.complex64)), np.complex64, (1,), device=True)
    X = dsp.to_device(x)
    out = DeviceArray((n, 1), np.complex64)
    step = c * 8
    for k in range(n // c):
        if k == 1:                                   # the first chunk also built the plan (one filter-transform launch)
            n0 = dsp.launch_count()
        xk = DeviceArray((c, 1), np.complex64, _base=X, _ptr=X.ptr + k * step)
        ok = DeviceArray((c, 1), np.complex64, _base=out, _ptr=out.ptr + k * step)
        dsp.fftfilt_(ok, f, xk)
    assert dsp.launch_count() - n0 == n // c - 1
    y = out.to_host()
    e_y, e_s = _relerr(y, yt), _relerr(f.state.to_host(), st)
    print(f"4097-tap ComplexF32 stream relerr: out {e_y:.3g}, state {e_s:.3g}")
    assert e_y < 2e-6 and e_s < 2e-6
    # against the stateless one-shot overlap-save of the whole signal (the headline kernel)
    one = DeviceArray((n, 1), np.complex64)
    plan = _lib.OsPlan(b, 0)
    plan.exec_dev(X.ptr, n, 1, one.ptr, n, 0)
    assert _relerr(y, one.to_host().astype(np.complex128)) < 2e-6
    plan.close()


# =============================================================================== GPU: edge cases and the C ABI

@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_edge_cases_and_host_form(dt):
    from dspb200 import device
    rng = np.random.default_rng(dt.num + 50)
    nb, nx, ncols = 300, 1000, 3
    b = _taps(rng, nb, dt)
    plan = _lib.OsPlan(b, 0)
    x, si = _ints(rng, (nx, ncols), dt, -8, 8), _ints(rng, (nb - 1, ncols), dt, -50, 50)
    X, SI = dsp.to_device(np.asfortranarray(x)), dsp.to_device(np.asfortranarray(si))
    full, tail, zfull, ztail = (_rint(a, dt) for a in _truth(b, x, si) + _truth(b, x, np.zeros_like(si)))

    def run(si_ptr, so):
        out = DeviceArray((nx, ncols), dt)
        plan.exec_state_dev(X.ptr, nx, ncols, si_ptr, so.ptr if so is not None else None, out.ptr, 0)
        device.sync()
        return out.to_host()

    SO = DeviceArray((nb - 1, ncols), dt)
    y = run(SI.ptr, SO)
    so = SO.to_host()
    assert np.array_equal(np.rint(y), full) and np.array_equal(np.rint(so), tail)
    y0 = run(None, SO)                                             # NULL si_in: a zero state
    assert np.array_equal(np.rint(y0), zfull) and np.array_equal(np.rint(SO.to_host()), ztail)
    y_nos = run(SI.ptr, None)                                      # NULL si_out: the state is discarded
    assert np.array_equal(np.rint(y_nos), np.rint(y)) and np.max(np.abs(y_nos - y)) <= _tol(dt)
    # the host form stages x and the state: it equals the device form bit for bit, and may filter in place
    xh, sh = np.asfortranarray(x.copy()), np.asfortranarray(si.copy())
    yh, soh = np.empty_like(xh), np.empty_like(sh)
    plan.exec_state(xh, nx, ncols, sh, soh, yh)
    assert np.array_equal(yh, y) and np.array_equal(soh, so)
    plan.exec_state(xh, nx, ncols, sh, sh, xh)                     # out is x, si_out is si_in
    assert np.array_equal(xh, y) and np.array_equal(sh, so)
    # nx == 0 passes the state through (and zeroes it from a NULL si_in)
    n0 = dsp.launch_count()
    S2 = DeviceArray((nb - 1, ncols), dt)
    plan.exec_state_dev(X.ptr, 0, ncols, SI.ptr, S2.ptr, X.ptr, 0)
    device.sync()
    assert np.array_equal(S2.to_host(), si) and dsp.launch_count() == n0
    plan.exec_state_dev(None, 0, ncols, None, S2.ptr, None, 0)
    device.sync()
    assert not np.any(S2.to_host())
    # the front end's empty chunk does no work and keeps the state
    f = dsp.DF2TFilter(dsp.PolynomialRatio(b, np.ones(1, dt)), dsp.to_device(si))
    assert dsp.fftfilt(f, DeviceArray((0, ncols), dt)).shape == (0, ncols)
    assert np.array_equal(f.state.to_host(), si) and dsp.launch_count() == n0
    plan.close()
    # nb == 1: no state, out = b[1] x, one launch
    p1 = _lib.OsPlan(np.array([3], dt), 0)
    out = DeviceArray((nx, ncols), dt)
    n0 = dsp.launch_count()
    p1.exec_state_dev(X.ptr, nx, ncols, None, None, out.ptr, 0)
    device.sync()
    assert np.array_equal(np.rint(out.to_host()), 3 * x) and dsp.launch_count() == n0 + 1
    g = dsp.DF2TFilter(dsp.PolynomialRatio(np.array([3], dt), np.ones(1, dt)), (ncols,), device=False)
    assert np.array_equal(np.rint(dsp.fftfilt(g, x.astype(g.state.dtype))), 3 * x)
    p1.close()


@pytest.mark.gpu
def test_overlap_refusals_launch_nothing():
    plan = _lib.OsPlan(np.ones(9), 0)
    dx = dsp.to_device(np.zeros((16, 2)))
    s, s2, o = DeviceArray((8, 2), np.float64), DeviceArray((8, 2), np.float64), DeviceArray((16, 2), np.float64)
    before = dsp.launch_count()
    with pytest.raises(_lib.DSPB200Error) as e:
        plan.exec_state_dev(dx.ptr, 16, 2, s.ptr, s.ptr + 8, o.ptr, 0)          # si_in with si_out
    assert e.value.code == _lib.EINVALID
    for x_ptr, out_ptr, si_out_ptr in ((dx.ptr, dx.ptr, s2.ptr), (dx.ptr, dx.ptr + 64, s2.ptr),
                                       (dx.ptr, o.ptr, dx.ptr + 8), (dx.ptr, o.ptr, o.ptr)):
        with pytest.raises(_lib.DSPB200Error, match="overlap") as e:          # x / out / state ranges may not overlap
            plan.exec_state_dev(x_ptr, 16, 2, s.ptr, si_out_ptr, out_ptr, 0)
        assert e.value.code == _lib.EINVALID
    with pytest.raises(_lib.DSPB200Error, match="overlap"):
        plan.exec_state_dev(dx.ptr, 16, 2, o.ptr + 8, s2.ptr, o.ptr, 0)        # si_in inside out
    assert dsp.launch_count() == before
    plan.exec_state_dev(dx.ptr, 16, 2, s.ptr, s2.ptr, o.ptr, 0)                  # disjoint buffers: one launch
    assert dsp.launch_count() == before + 1
    plan.close()
    # a plan with an explicit fused nfft below 1024 has no stateful kernel: refused, not run another way
    small = _lib.OsPlan(np.ones(9), 256)
    before = dsp.launch_count()
    with pytest.raises(_lib.DSPB200Error) as e:
        small.exec_state_dev(dx.ptr, 16, 2, s.ptr, s2.ptr, o.ptr, 0)
    assert e.value.code == _lib.EUNSUPPORTED and dsp.launch_count() == before
    small.close()
