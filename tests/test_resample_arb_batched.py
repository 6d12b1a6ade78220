"""Arbitrary-rate resampling of many channels in one launch (resample_arb_batch_kernel, csrc/resample.cu).

`arb_tiling` restates the host's tile sizing (rs_arb_tiling), so the CPU tests can check with exact rational phases that
every output's window lies inside the span its tile stages in shared memory, and that a CTA's shared memory fits an H100.
A second CPU test replaces the device plan with a numpy model and checks the arguments `resample` passes for matrices and
3-D arrays.

The main GPU check is exact.  Taps are integers in [-4, 4], samples integers in [-8, 8] (both parts for complex input),
acc0 = 0 and delta a dyadic rational with two fractional bits, so every phase fraction alpha has two bits.  Each dot product
is then an integer below 2^24 in magnitude and each output yu*alpha + yl a multiple of 1/4 below 2^22: exact in Float32.
Every output must equal the float64 closed form bit for bit, whatever the tile, span or bank placement.

These exact checks cover only acc0 = 0 and dyadic phases.  tests/test_resample_arb_kernel_paths.py checks every instance
and entry point against exact phases for any acc0 and delta (non-dyadic rates, phases on and beside phase boundaries,
j*delta past 2^31), within a proven phase bound; the checks here stay as the bit-exact special case."""
import math
from fractions import Fraction

import numpy as np
import pytest

import dspb200 as dsp
from conftest import relerr
from oracle import filters as of

F32, F64, C64, C128 = (np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))
# the six (input, taps) combinations that select distinct instances in rs_arb_run
TRIPLES = ((F32, F32), (F32, F64), (F64, F64), (C64, F32), (C64, F64), (C128, F64))
SMEM_OPTIN = 227 * 1024          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
SPAN_MAX = BANKS_MAX = 96 * 1024  # RS_ARB_SPAN_MAX, RS_ARB_BANKS_MAX
RATES = (0.98, 1.0001, 1.2957, 2.618, 0.7312, 1 / 55.55)


# =============================================================================== tile sizing restated from rs_arb_tiling

def arb_tiling(tpp, nphi, delta, x_bytes, tap_bytes):
    """(tile, threads, xs_len, banks_in_smem, smem bytes) as rs_arb_tiling computes them."""
    bank_bytes = 2 * nphi * tpp * tap_bytes
    banks = bank_bytes <= BANKS_MAX
    V = 16 // x_bytes
    tile, xs_len = 256, 0
    for T in (1024, 512, 256, 128, 64, 32):
        steps = math.ceil((T - 1) * delta / nphi)          # same double expression as the C++ code
        if steps * x_bytes > SPAN_MAX:
            continue
        span = steps + tpp + 1
        n = (span + V - 1 + V - 1) // V * V
        if n * x_bytes > SPAN_MAX:
            continue
        tile, xs_len = T, n
        break
    return tile, min(tile, 256), xs_len, banks, xs_len * x_bytes + (bank_bytes if banks else 0)


def _sizes(dtype_x, dtype_h):
    x = np.dtype(dtype_x)
    tr = 8 if x in (F64, C128) or np.dtype(dtype_h) == F64 else 4
    return x.itemsize, tr


def _undelayed(h, rate, nphi):
    """(n0, acc0, delta) of a fresh FIRArbitrary filter after undelay!, from the literal oracle."""
    so = of.FIRArbitraryState(h, rate, nphi)
    so.setphase(so.timedelay())
    return so.input_deficit - 1, so.acc, so.delta, so


def _exact_q(acc0, delta, nphi, js):
    """floor((acc0 + j*delta) / Nphi) in exact rational arithmetic."""
    A, D = Fraction(acc0), Fraction(delta)
    den = A.denominator * D.denominator // math.gcd(A.denominator, D.denominator)
    an, dn = A.numerator * (den // A.denominator), D.numerator * (den // D.denominator)
    return [(an + j * dn) // (nphi * den) for j in js]


@pytest.mark.parametrize("nphi", [1, 32, 128])
@pytest.mark.parametrize("rate", RATES)
def test_tile_spans_hold_every_window(rate, nphi):
    cases = 0
    for taps in ("default", "short"):
        h = dsp.resample_filter(rate, nphi) if taps == "default" else np.ones(max(3, nphi // 2 + 2))
        tpp = -(-h.size // nphi)
        _, acc0, delta, _ = _undelayed(h, rate, nphi)
        for dx, dh in TRIPLES:
            xb, tb = _sizes(dx, dh)
            tile, threads, xs_len, banks, smem = arb_tiling(tpp, nphi, delta, xb, tb)
            assert smem <= SMEM_OPTIN and threads == min(tile, 256)
            if xs_len == 0:
                continue
            V = 16 // xb
            ntiles = 6
            q = _exact_q(acc0, delta, nphi, range(ntiles * tile))
            for k in range(ntiles):
                qt = q[k * tile:(k + 1) * tile]
                # the kernel floors the span start to a multiple of V: up to V - 1 extra samples in front
                for shift in (0, V - 1):
                    start = qt[0] - (tpp - 1) - shift
                    for qj in qt:                              # window of output j: [qj - (tpp-1), qj]
                        assert qj - (tpp - 1) >= start and qj + 1 <= start + xs_len, (rate, nphi, taps, dx, dh, k)
            cases += 1
    assert cases > 0


def test_tiling_reaches_both_bank_placements_and_small_tiles():
    seen = set()
    for rate in RATES:
        h = dsp.resample_filter(rate, 32)
        tpp = -(-h.size // 32)
        for dx, dh in TRIPLES:
            tile, _, xs_len, banks, _ = arb_tiling(tpp, 32, 32 / rate, *_sizes(dx, dh))
            seen.add((banks, tile < 256, xs_len > 0))
    assert (True, False, True) in seen and (False, False, True) in seen and (False, True, True) in seen


# =============================================================================== host bookkeeping with a numpy kernel

class _ModelPlan:
    """numpy model of the arbitrary-rate kernel's contract; records the batched calls."""
    calls = []

    def __init__(self, dtype_x, h, nphases):
        self.h, self.n = np.asarray(h, dtype=np.float64), int(nphases)
        self.out_dtype = np.result_type(np.dtype(dtype_x), np.asarray(h).dtype)
        self.pfb = of.taps2pfb(self.h, self.n)
        self.dpfb = of.taps2pfb(np.concatenate([np.diff(self.h), [0.0]]), self.n)

    def _column(self, xc, nx, n0, acc0, delta, nout):
        tpp = self.pfb.shape[0]
        y = np.empty(nout, dtype=np.result_type(self.out_dtype, np.float64))
        for j in range(nout):
            P = Fraction(acc0) + j * Fraction(delta)
            q = P // self.n
            r = float(P - q * self.n)
            phi, alpha = int(np.floor(r)), r - np.floor(r)
            first = n0 + int(q) - (tpp - 1)
            win = np.array([xc[i] if 0 <= i < nx else 0.0 for i in range(first, first + tpp)])
            y[j] = np.dot(self.dpfb[:, phi], win) * alpha + np.dot(self.pfb[:, phi], win)
        return y

    def exec(self, x, nx, n0, acc0, delta, out, nout):
        out[:nout] = self._column(x, nx, n0, acc0, delta, nout)

    def exec_batch(self, x, nx, ldx, ncols, n0, acc0, delta, out, nout):
        assert x.flags.f_contiguous and x.shape == (ldx, ncols) and out.shape == (nout, ncols)
        _ModelPlan.calls.append(dict(nx=nx, ldx=ldx, ncols=ncols, n0=n0, acc0=acc0, delta=delta, nout=nout))
        for c in range(ncols):
            out[:, c] = self._column(x[:, c], nx, n0, acc0, delta, nout)

    def close(self):
        pass


def test_matrix_resample_passes_one_batched_call(monkeypatch):
    from dspb200 import _lib
    monkeypatch.setattr(_lib, "ResampleArbPlan", _ModelPlan)
    rng = np.random.default_rng(11)
    for rate in (0.7312, 1.2957, 2.618, 1 / 55.55):
        h = dsp.resample_filter(rate, 32)
        n0, acc0, delta, so = _undelayed(h, rate, 32)
        for shape, dims in (((120, 3), 0), ((4, 120), 1), ((120, 2, 3), 0), ((2, 120, 3), 1), ((2, 3, 120), 2)):
            x = rng.standard_normal(shape)
            _ModelPlan.calls.clear()
            y = dsp.resample(x, rate, dims=dims)
            outlen = math.ceil(120 * rate)
            npad = so.inputlength(outlen, round_up=True) + 1
            assert len(_ModelPlan.calls) == 1
            c = _ModelPlan.calls[0]
            assert c == dict(nx=min(120, npad), ldx=120, ncols=x.size // 120, n0=n0, acc0=acc0, delta=delta, nout=outlen)
            xm = np.moveaxis(x, dims, 0)
            assert y.shape == tuple(outlen if a == dims else s for a, s in enumerate(shape))
            ym = np.moveaxis(y, dims, 0)
            for idx in np.ndindex(xm.shape[1:]):
                col = xm[(slice(None),) + idx]
                assert np.array_equal(ym[(slice(None),) + idx], dsp.resample(np.ascontiguousarray(col), rate))
            assert np.allclose(ym[(slice(None),) + (0,) * (x.ndim - 1)],
                               of.resample_arb_literal(xm[(slice(None),) + (0,) * (x.ndim - 1)], rate), rtol=1e-9, atol=1e-12)


# =============================================================================== GPU: exact against the closed form

def _int_signal(rng, shape, dt):
    v = rng.integers(-8, 9, shape).astype(np.float64)
    if np.dtype(dt).kind == "c":
        v = v + 1j * rng.integers(-8, 9, shape)
    return v.astype(dt)


def closed_form(x, nx, h, nphi, n0, delta, nout, out_dtype):
    """Exact outputs for acc0 = 0 and a dyadic delta: x is (ldx, ncols); samples outside [0, nx) are zero."""
    x = np.asarray(x)[:nx]
    ncols = x.shape[1]
    w = np.complex128 if np.iscomplexobj(x) else np.float64
    h = np.asarray(h, dtype=np.float64)
    pfb = of.taps2pfb(h, nphi)
    dpfb = of.taps2pfb(np.concatenate([np.diff(h), [0.0]]), nphi)
    tpp = pfb.shape[0]
    P = np.arange(nout, dtype=np.float64) * delta                # exact: small dyadic multiples
    q = np.floor(P / nphi)
    r = P - q * nphi
    phi = np.floor(r).astype(np.int64)
    alpha = r - phi
    newest = n0 + q.astype(np.int64)
    xpad = np.zeros((nx + 2 * tpp, ncols), dtype=w)              # xpad[s + tpp] = x[s]
    xpad[tpp:tpp + nx] = x
    yl = np.zeros((nout, ncols), dtype=w)
    yu = np.zeros((nout, ncols), dtype=w)
    for t in range(tpp):
        s = newest - (tpp - 1) + t
        ok = (s >= 0) & (s < nx)
        v = np.where(ok[:, None], xpad[np.clip(s, -tpp, nx + tpp - 1) + tpp], 0)
        yl += pfb[t, phi][:, None] * v
        yu += dpfb[t, phi][:, None] * v
    return (yu * alpha[:, None] + yl).astype(out_dtype)


def _run_exact(dx, dh, nphi, hlen, nx, ldx, ncols, n0, delta, nout, offset=0, seed=0, host=False):
    rng = np.random.default_rng(seed)
    h = rng.integers(-4, 5, hlen).astype(dh)
    x = _int_signal(rng, (ldx, ncols), dx)
    plan = dsp._lib.ResampleArbPlan(dx, h, nphi)
    want = closed_form(x, nx, h, nphi, n0, delta, nout, plan.out_dtype)
    if host:
        got = np.empty((nout, ncols), dtype=plan.out_dtype, order="F")
        plan.exec_batch(np.asfortranarray(x), nx, ldx, ncols, n0, 0.0, delta, got, nout)
    else:
        # `offset` elements in front shift the column base off its 16-byte alignment
        buf = np.zeros(ldx * ncols + offset, dtype=dx)
        buf[offset:] = np.asfortranarray(x).ravel(order="F")
        dxa = dsp.to_device(buf)
        dout = dsp.DeviceArray((nout, ncols), plan.out_dtype)
        plan.exec_batch_dev(dxa.ptr + offset * np.dtype(dx).itemsize, nx, ldx, ncols, n0, 0.0, delta, dout.ptr, nout, 0)
        got = dout.to_host()
    plan.close()
    assert got.dtype == want.dtype
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{len(bad)} outputs differ, first at {bad[:4].tolist()}"


@pytest.mark.gpu
@pytest.mark.parametrize("dx,dh", TRIPLES, ids=[f"{a}-{b}" for a, b in TRIPLES])
@pytest.mark.parametrize("nphi", [1, 32])
def test_exact_against_closed_form(dx, dh, nphi):
    hlen = 21 if nphi == 1 else 39 * 32 - 7                     # 21 / 39 taps per phase
    tpp = -(-hlen // nphi)
    for delta in (12.25, 31.75, 32.5, 40.5, 1777.5):
        d = delta / 32 * nphi if nphi == 1 else delta             # Nphi = 1: about the same rates
        nout = 5000 if delta < 100 else 900                        # several tiles
        nx = int(nout * d / nphi) + 3
        # windows straddle both ends: n0 < tpp - 1 at the start, and the last outputs run past nx
        _run_exact(dx, dh, nphi, hlen, nx, nx, 3, 5, d, nout + 2 * int(tpp * nphi / d + 1), seed=int(delta * 4))
    # a column stride that is not a multiple of 16 bytes, ldx > nx, an unaligned base, and the host entry
    _run_exact(dx, dh, nphi, hlen, 1001, 1003, 3, tpp + 3, 32.5, 1100, offset=1, seed=3)
    _run_exact(dx, dh, nphi, hlen, 1001, 1003, 3, tpp + 3, 32.5, 1100, seed=4, host=True)
    # nx < tpp, nx = 0, one column, no columns
    _run_exact(dx, dh, nphi, hlen, tpp - 2, tpp - 2, 1, 2, 31.75, 40, seed=5)
    _run_exact(dx, dh, nphi, hlen, 0, 0, 2, 0, 31.75, 40, seed=6)
    _run_exact(dx, dh, nphi, hlen, 300, 300, 0, 0, 31.75, 40, seed=7)


@pytest.mark.gpu
def test_exact_many_short_columns():
    # more columns than a grid dimension holds
    _run_exact(F32, F32, 32, 32 * 3, 7, 7, 70000, 1, 40.5, 6, seed=8)
    _run_exact(C64, F64, 32, 32 * 3, 6, 9, 66000, 2, 12.25, 9, seed=9)


@pytest.mark.gpu
@pytest.mark.parametrize("dx,dh", TRIPLES, ids=[f"{a}-{b}" for a, b in TRIPLES])
def test_exact_long_taps_banks_in_global_memory(dx, dh):
    hlen = 32 * 400                                              # 400 taps per phase: both banks > 96 KB
    assert not arb_tiling(400, 32, 40.5, *_sizes(dx, dh))[3]
    _run_exact(dx, dh, 32, hlen, 3000, 3000, 2, 50, 40.5, 2500, seed=10)
    _run_exact(dx, dh, 32, hlen, 3000, 3001, 2, 50, 1777.5, 60, offset=1, seed=11)


# =============================================================================== GPU: public API

def _randn(rng, shape, dt):
    v = rng.standard_normal(shape)
    if np.dtype(dt).kind == "c":
        v = v + 1j * rng.standard_normal(shape)
    return v.astype(dt)


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [0.7312, 1.2957, 2.618, 1 / 55.55])
@pytest.mark.parametrize("dt", [F32, F64, C64, C128], ids=str)
def test_matrix_columns_equal_vector_calls(rate, dt):
    rng = np.random.default_rng(21)
    X = _randn(rng, (700, 5), dt)
    Y = dsp.resample(X, rate, dims=0)
    assert Y.shape == (math.ceil(700 * rate), 5)
    for c in range(5):
        assert np.array_equal(Y[:, c], dsp.resample(X[:, c], rate))
    tol = 2e-6 if dt in (F32, C64) else 1e-10
    assert relerr(Y[:, 0], of.resample_arb_literal(X[:, 0], rate)) < tol
    assert np.array_equal(dsp.resample(np.ascontiguousarray(X.T), rate, dims=1), Y.T)
    X3 = X[:, :4].reshape(700, 2, 2)
    Y3 = dsp.resample(np.moveaxis(X3, 0, 2), rate, dims=2)
    assert np.array_equal(np.moveaxis(Y3, 2, 0).reshape(-1, 4), Y[:, :4])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F64, C64, C128], ids=str)
def test_device_arrays_stay_on_the_device(dt):
    rng = np.random.default_rng(22)
    X = _randn(rng, (3001, 6), dt)
    for rate in (0.7312, 2.618, 1 / 55.55, Fraction(3, 2), Fraction(2, 7), 3):
        for x in (X[:, 0].copy(), X):
            d = dsp.resample(dsp.to_device(x), rate, dims=0 if x.ndim == 2 else None)
            assert isinstance(d, dsp.DeviceArray)
            want = dsp.resample(x, rate, dims=0 if x.ndim == 2 else None)
            got = d.to_host()
            assert got.shape == want.shape and got.dtype == want.dtype and np.array_equal(got, want), rate
    with pytest.raises(dsp.ArgumentError):
        dsp.resample(dsp.to_device(X), 0.7312, dims=1)
    with pytest.raises(dsp.ArgumentError):
        dsp.resample(dsp.to_device(X), Fraction(3, 2), dims=1)


@pytest.mark.gpu
def test_one_launch_for_64_columns():
    X = np.random.default_rng(23).standard_normal((5000, 64)).astype(np.float32)
    dsp.resample(X, 0.9802414928649835, dims=0)                 # warm-up
    n = dsp.launch_count()
    dsp.resample(X, 0.9802414928649835, dims=0)
    assert dsp.launch_count() - n == 1
    D = dsp.to_device(X)
    n = dsp.launch_count()
    dsp.resample(D, 0.9802414928649835, dims=0)
    assert dsp.launch_count() - n == 1


@pytest.mark.gpu
def test_full_size_probe_64_channels():
    rate, nphi = 0.9802414928649835, 32
    h = dsp.resample_filter(rate, nphi).astype(np.float32)
    nx, nchan = 1 << 20, 64
    X = np.random.default_rng(24).standard_normal((nx, nchan), dtype=np.float32)
    Y = dsp.resample(dsp.to_device(X), rate, h, dims=0).to_host()
    outlen = math.ceil(nx * rate)
    assert Y.shape == (outlen, nchan) and Y.dtype == np.float32
    n0, acc0, delta, so = _undelayed(h, rate, nphi)
    npad = so.inputlength(outlen, round_up=True) + 1
    m = min(nx, npad)
    tpp = -(-h.size // nphi)
    tile = arb_tiling(tpp, nphi, delta, 4, 4)[0]
    js = sorted(set(list(range(40)) + list(range(outlen - 40, outlen)) + list(range(outlen // 2 - 20, outlen // 2 + 20))
                    + [k * tile + d for k in (1, 7, 333, outlen // tile - 1) for d in (-2, -1, 0, 1)]))
    pfb = of.taps2pfb(h.astype(np.float64), nphi)
    dpfb = of.taps2pfb(np.concatenate([np.diff(h), [np.float32(0)]]).astype(np.float64), nphi)
    q = _exact_q(acc0, delta, nphi, js)
    A, D = Fraction(acc0), Fraction(delta)
    for c in (0, 17, 63):
        want = np.empty(len(js))
        for k, j in enumerate(js):
            r = float(A + j * D - q[k] * nphi)
            phi = int(math.floor(r))
            first = n0 + q[k] - (tpp - 1)
            win = np.array([float(X[i, c]) if 0 <= i < m else 0.0 for i in range(first, first + tpp)])
            want[k] = np.dot(dpfb[:, phi], win) * (r - phi) + np.dot(pfb[:, phi], win)
        assert relerr(Y[js, c], want) < 2e-6, c
