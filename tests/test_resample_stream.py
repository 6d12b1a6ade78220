"""Streaming FIRFilter on the device (FIRFilter(h, ratio, nphases, device=True)): chunked vectors and len x nchan matrices
through dspb200_resample_stream_exec_dev / dspb200_resample_arb_stream_exec_dev.

A call filters the virtual column [history; x] of every channel.  The rational kinds run the first j_seam outputs (the ones
whose window reaches into the history) and the new history in one edge kernel, then the rest through the kernel family
rs_launch picks, on the chunk alone; the arbitrary-rate kernel reads the virtual column itself.  The host form
(concatenation, one launch per channel) and the device form share the per-call bookkeeping `FIRFilter._step`.

CPU tests: the bookkeeping against the literal reference loops, j_seam against a brute-force count, and the argument,
residency and overlap rules with a numpy stand-in for the library.  GPU tests: exact on integer data (taps in [-4, 4],
samples in [-8, 8]) for every rational kernel family, device against host chunk by chunk and history by history, the
arbitrary rate in all six type combinations, launch counts and the C ABI's refusals."""
import math
from fractions import Fraction

import numpy as np
import pytest

import dspb200 as dsp
from dspb200 import _lib
from dspb200.device import DeviceArray
from oracle import filters as of
from test_resample_kernel_paths import (C64, C128, F32, F64, expected_family, int_signal, int_taps, mp2_v3,
                                        polyphase_ref, tile_outputs)

ARB_TRIPLES = ((F32, F32), (F32, F64), (F64, F64), (C64, F32), (C64, F64), (C128, F64))
# one case per rational kernel family (mp2 with both tap sources, mp, tiled, generic) and per FIRFilter kind
STREAM_CASES = [(3, 2, 38, F32, F32), (2, 3, 25, F32, F64), (2, 1, 129, C64, F32), (5, 2, 51, C64, F32),
                (11, 5, 40, F64, F64), (1, 1, 33, F32, F32), (1, 3, 31, F64, F64)]


def _kind(I, D):
    return "standard" if I == D == 1 else "interpolator" if D == 1 else "decimator" if I == 1 else "rational"


def _case_id(c):
    I, D, hlen, tx, th = c
    return f"{I}/{D}-{tx.name}-{th.name}-h{hlen}-{expected_family(I, D, hlen, tx, th)}"


def _chunks(rng, n, sizes):
    """Split range(n) into consecutive chunks whose lengths cycle through `sizes` (None: random lengths)."""
    out, a, k = [], 0, 0
    while a < n:
        c = int(rng.integers(0, 40)) if sizes is None else sizes[k % len(sizes)]
        out.append((a, min(n, a + c)))
        a, k = a + c, k + 1
    return out


# =============================================================================== CPU: bookkeeping

def _oracle_state(kind, h, ratio, nphases):
    return of.FIRArbitraryState(h, ratio, nphases) if kind == "arbitrary" else of.FIRFilterState(h, ratio)


@pytest.mark.parametrize("ratio", [1, 3, Fraction(1, 3), Fraction(3, 2), Fraction(4, 7), 0.98, 1.37])
def test_step_matches_reference_loops(ratio):
    rng = np.random.default_rng(5)
    arb = isinstance(ratio, float)
    h = rng.standard_normal(3 * 32 + 5 if arb else 23)
    for taus in ([], [0.4], [2.6], [9.3]):
        if ratio == 1 and taus:
            continue                          # the literal single-rate loop does not consume a phase shift
        f = dsp.FIRFilter(h, ratio, 32)
        ref = _oracle_state(f.kind, h, ratio, 32)
        for t in taus:
            f.setphase(t)
            ref.setphase(t)
        sizes = [0, 1, 0, 2, 1, 1, 17, 0, 3, 60, 1, 5] + [int(v) for v in rng.integers(0, 30, 12)]
        for xlen in sizes:
            st = f._step(f.phi_idx, f.input_deficit, f.phi_accumulator, xlen)
            y = ref.filt(rng.standard_normal(xlen))
            f._commit(st)
            assert st.nout == y.size, (ratio, taus, xlen)
            assert (f.phi_idx, f.input_deficit) == (ref.phi_idx, ref.input_deficit), (ratio, taus, xlen)
            if arb:
                assert f.phi_accumulator == pytest.approx(ref.acc, abs=1e-9)


@pytest.mark.parametrize("ratio", [Fraction(3, 2), Fraction(2, 3), 4, Fraction(1, 4), Fraction(7, 3), 1])
def test_j_seam_counts_outputs_that_read_the_history(ratio):
    for hlen in (1, 5, 24, 37):
        for tau in (None, 0.0, 0.7, 1.5, 3.2, 12.0, 40.0):
            if tau is not None and ratio == 1:
                continue
            f = dsp.FIRFilter(np.ones(hlen), ratio)
            if tau is not None:
                f.setphase(tau)
            I, D, H = f.interpolation, f.decimation, f.history_len
            tpp = H + 1
            for xlen in (0, 1, 2, H, H + 1, 3 * H + 7, 200):
                st = f._step(f.phi_idx, f.input_deficit, f.phi_accumulator, xlen)
                oldest = [st.n0 + (st.phase0 + j * D) // I - (tpp - 1) for j in range(st.nout)]
                assert st.j_seam == sum(o < H for o in oldest), (ratio, hlen, tau, xlen)
                assert all(o >= 0 for o in oldest)
                if st.nout:
                    assert st.n0 + (st.phase0 + (st.nout - 1) * D) // I <= H + xlen - 1 or f.kind == "standard"
            # deficits past H + 1 leave no output in the seam
            if f.input_deficit > H + 1:
                assert f._step(f.phi_idx, f.input_deficit, 0.0, 500).j_seam == 0


# =============================================================================== CPU: argument rules with a stand-in library

class _FakePlan:
    """numpy model of a resample plan: exec / stream_exec_dev record their calls; exec computes the polyphase sum."""
    calls = []

    def __init__(self, dtype_x, h, interp, decim=None):
        self.h, self.I, self.D = np.asarray(h), int(interp), 1 if decim is None else int(decim)
        dx = np.dtype(dtype_x)
        f64 = dx in (F64, C128) or self.h.dtype == F64
        self.out_dtype = np.dtype((np.complex128 if f64 else np.complex64) if dx.kind == "c" else (np.float64 if f64 else np.float32))

    def exec(self, xe, nx, *args):
        if len(args) == 5:                        # rational: (ncols, n0, phi0, out, nout)
            _, n0, phi0, out, nout = args
            out[:] = polyphase_ref(xe, self.h, self.I, self.D, n0, phi0, nout)
        _FakePlan.calls.append(("exec", nx))

    def stream_exec_dev(self, *args):
        _FakePlan.calls.append(("stream",) + args)

    def close(self):
        pass


class _AddressOnly(DeviceArray):
    """A DeviceArray at a dummy address: nothing is allocated, read or launched.  New arrays get fresh addresses."""
    _next = [1 << 30]

    def __init__(self, shape, dtype, _base=None, _ptr=None):
        if _ptr is None:
            _ptr = _AddressOnly._next[0]
            _AddressOnly._next[0] += 1 << 20
        super().__init__(shape, dtype, _base=_base, _ptr=_ptr)


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(_lib, "ResamplePlan", _FakePlan)
    monkeypatch.setattr(_lib, "ResampleArbPlan", _FakePlan)
    monkeypatch.setattr(dsp.filters, "DeviceArray", _AddressOnly)
    _FakePlan.calls = []
    return _FakePlan


def test_stream_cases_reach_every_family():
    fams = {(expected_family(*c), mp2_v3(*c[:2], *c[3:]) if expected_family(*c) == "mp2" else None) for c in STREAM_CASES}
    assert fams == {("mp2", True), ("mp2", False), ("mp", None), ("tiled", None), ("generic", None)}
    assert {_kind(*c[:2]) for c in STREAM_CASES} == {"standard", "interpolator", "decimator", "rational"}
    assert all(expected_family(*c, ncols=70) == expected_family(*c) for c in STREAM_CASES)


def test_residency_and_argument_rules_fail_before_any_launch(fake):
    h = np.arange(1.0, 12.0)
    host = dsp.FIRFilter(h, Fraction(3, 2))
    dx = _AddressOnly((40, 3), np.float64, _ptr=4096)
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(host, dx)
    with pytest.raises(dsp.ArgumentError):
        dsp.filt_(_AddressOnly((80,), np.float64), host, np.zeros(40))
    dev = dsp.FIRFilter(h, Fraction(3, 2), device=True)
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(dev, np.zeros(40))
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(dev, _AddressOnly((4, 2, 2), np.float64))
    assert fake.calls == [] and dev._dev_key is None
    y = dsp.filt(dev, dx)                                  # first chunk: fixes Float64 x 3 channels
    assert isinstance(y, DeviceArray) and y.shape == (60, 3) and y.dtype == np.float64
    (call,) = fake.calls
    hist_in, hist_out, xp, nx, nch, deficit, phi0, outp, ldo, nout = call[1:11]
    assert hist_in is None and (xp, nx, nch, deficit, phi0, outp, ldo, nout) == (4096, 40, 3, 1, 0, y.ptr, 60, 60)
    state = (dev.phi_idx, dev.input_deficit)
    for bad in (_AddressOnly((40, 3), np.float32), _AddressOnly((40, 4), np.float64), _AddressOnly((40,), np.float64)):
        with pytest.raises(dsp.ArgumentError):
            dsp.filt(dev, bad)
    st = dev._step(dev.phi_idx, dev.input_deficit, 0.0, 40)
    x2 = _AddressOnly((40, 3), np.float64, _ptr=1 << 24)
    for buf in (_AddressOnly((st.nout - 1, 3), np.float64),              # too short
                _AddressOnly((st.nout, 3), np.float32),                  # wrong eltype
                _AddressOnly((st.nout, 2), np.float64),                  # wrong channel count
                _AddressOnly((st.nout, 3), np.float64, _ptr=(1 << 24) + 8 * 100),   # overlaps x
                _AddressOnly((st.nout, 3), np.float64, _ptr=(1 << 24) - 8 * st.nout * 3 + 8)):
        with pytest.raises(dsp.ArgumentError):
            dsp.filt_(buf, dev, x2)
    with pytest.raises(dsp.ArgumentError):
        dsp.filt_(np.zeros((st.nout, 3)), dev, x2)
    assert len(fake.calls) == 1 and (dev.phi_idx, dev.input_deficit) == state
    # a longer buffer: ldo is its row count, the return value the number of outputs
    buf = _AddressOnly((st.nout + 5, 3), np.float64)
    assert dsp.filt_(buf, dev, x2) == st.nout
    c2 = fake.calls[-1]
    assert c2[1] == hist_out and c2[8:11] == (buf.ptr, st.nout + 5, st.nout)          # histories swap
    assert dev.history.ptr == c2[2]
    # empty chunk: nothing launched, state unchanged; short chunk after setphase: history only
    n = len(fake.calls)
    assert dsp.filt(dev, _AddressOnly((0, 3), np.float64)).shape == (0, 3) and len(fake.calls) == n
    dev.setphase(5.0)
    d0 = dev.input_deficit
    assert dsp.filt(dev, _AddressOnly((2, 3), np.float64)).shape == (0, 3)
    assert len(fake.calls) == n + 1 and fake.calls[-1][10] == 0 and dev.input_deficit == d0 - 2
    # reset() drops the eltype, channel count and history
    dev.reset()
    assert dev._dev_key is None and dev.history is None and (dev.phi_idx, dev.input_deficit) == (1, 1)
    dsp.filt(dev, _AddressOnly((7,), np.complex64))
    assert fake.calls[-1][1] is None and dev.history.shape == (dev.history_len,)


def test_host_filt_buffer_and_routing(fake):
    rng = np.random.default_rng(3)
    h, x = int_taps(rng, 23, F64), int_signal(rng, 90, F64)
    f, g = dsp.FIRFilter(h, Fraction(2, 3)), dsp.FIRFilter(h, Fraction(2, 3))
    want = dsp.filt(f, x[:50])
    st = g._step(g.phi_idx, g.input_deficit, 0.0, 50)
    with pytest.raises(dsp.ArgumentError):
        dsp.filt_(np.zeros(st.nout - 1), g, x[:50])
    assert (g.phi_idx, g.input_deficit, g.history) == (1, 1, None)
    buf = np.full(st.nout + 3, 7.0)
    assert dsp.filt_(buf, g, x[:50]) == st.nout == want.size
    assert np.array_equal(buf[:st.nout], want) and np.all(buf[st.nout:] == 7.0)
    assert np.array_equal(dsp.filt(f, x[50:]), dsp.filt(g, x[50:]))
    with pytest.raises(dsp.ArgumentError):
        dsp.filt(f, x, 2)


# =============================================================================== GPU

def _dev_matrix(x):
    return dsp.to_device(np.asfortranarray(x))


def _exact(y, ref):
    return np.array_equal(y.astype(np.complex128 if y.dtype.kind == "c" else np.float64), ref)


@pytest.mark.gpu
@pytest.mark.parametrize("I,D,hlen,tx,th", STREAM_CASES, ids=[_case_id(c) for c in STREAM_CASES])
def test_rational_stream_exact_every_family(I, D, hlen, tx, th):
    rng = np.random.default_rng(hlen)
    h = int_taps(rng, hlen, th)
    H = -(-hlen // I) - 1
    tile_in = max(2, tile_outputs(expected_family(I, D, hlen, tx, th), I, D, tx, th) * D // I)
    kinds_with_phase = _kind(I, D) != "standard"
    for nch in (3, 70):
        for sizes in ([1], [2], [max(H - 1, 1)], [max(H, 1)], [H + 1], [tile_in - 1], [tile_in + 1], None):
            for tau in ((None, 3.7, H + 4.5) if kinds_with_phase else (None,)):
                if tau is not None and (nch == 70 or sizes not in ([1], [H + 1], None)):
                    continue
                n = 2 * tile_in + 5 if sizes is not None and sizes[0] >= tile_in - 1 else 3 * H + 300
                x = int_signal(rng, (n, nch), tx)
                f = dsp.FIRFilter(h, Fraction(I, D), device=True)
                hosts = [dsp.FIRFilter(h, Fraction(I, D)) for _ in (0, nch - 1)]
                if tau is not None:
                    for g in [f] + hosts:
                        g.setphase(tau)
                n0, phi0 = f.input_deficit - 1, (f.phi_idx - 1 if _kind(I, D) in ("rational", "interpolator") else 0)
                parts = []
                for a, b in _chunks(rng, n, sizes):
                    y = f.filt(_dev_matrix(x[a:b])).to_host()
                    parts.append(y)
                    for g, c in zip(hosts, (0, nch - 1)):
                        assert np.array_equal(g.filt(x[a:b, c]), y[:, c]), (nch, sizes, tau, a)
                        if f.history is not None:
                            assert np.array_equal(f.history.to_host()[:, c], g.history), (nch, sizes, tau, a)
                y = np.concatenate(parts)
                if _kind(I, D) != "standard" or tau is None:
                    assert _exact(y, polyphase_ref(x, h, I, D, n0, phi0, y.shape[0])), (nch, sizes, tau)


@pytest.mark.gpu
def test_rational_stream_70000_channels():
    rng = np.random.default_rng(70)
    h = int_taps(rng, 38, F32)
    nch, n = 70000, 45
    x = int_signal(rng, (n, nch), F32)
    f = dsp.FIRFilter(h, Fraction(3, 2), device=True)
    parts = [f.filt(_dev_matrix(x[a:a + 5])).to_host() for a in range(0, n, 5)]
    y = np.concatenate(parts)
    assert y.shape == (math.ceil(n * 1.5), nch)
    assert _exact(y, polyphase_ref(x, h, 3, 2, 0, 0, y.shape[0]))
    assert np.array_equal(f.history.to_host(), x[n - f.history_len:])


@pytest.mark.gpu
def test_vector_chunks_and_buffer_rows():
    rng = np.random.default_rng(8)
    h = int_taps(rng, 38, F64)
    x = int_signal(rng, 300, F64)
    f, g = dsp.FIRFilter(h, Fraction(3, 2), device=True), dsp.FIRFilter(h, Fraction(3, 2))
    big = dsp.to_device(np.full(400, -99.0))
    most = 0
    for a, b in ((0, 10), (10, 11), (11, 200), (200, 300)):
        want = g.filt(x[a:b])
        assert dsp.filt_(big, f, dsp.to_device(x[a:b])) == want.size
        got = big.to_host()
        assert np.array_equal(got[:want.size], want)
        most = max(most, want.size)
        assert dsp.filt(f, dsp.to_device(x[:0])).shape == (0,)
    assert most < 400 and np.all(got[most:] == -99.0)


def _arb_views(x, aligned, rng, sizes):
    """Chunks of x (n x nch) as DeviceArray views into one buffer: chunk bases 16-byte aligned with 16-byte column strides
    (cp.async staging) or at odd element offsets."""
    n, nch = x.shape
    bounds = _chunks(rng, n, sizes)
    esz = x.dtype.itemsize
    offs, pos = [], 0
    for a, b in bounds:
        pos += 0 if aligned else 1
        offs.append(pos)
        pos += (b - a) * nch
        pos = -(-pos * esz // 64) * 64 // esz
    flat = np.zeros(pos + 8, dtype=x.dtype)
    for (a, b), o in zip(bounds, offs):
        flat[o:o + (b - a) * nch] = np.asfortranarray(x[a:b]).ravel(order="F")
    buf = dsp.to_device(flat)
    return buf, [((a, b), DeviceArray((b - a, nch), x.dtype, _base=buf, _ptr=buf.ptr + o * esz)) for (a, b), o in zip(bounds, offs)]


@pytest.mark.gpu
@pytest.mark.parametrize("tx,th", ARB_TRIPLES, ids=[f"{a.name}-{b.name}" for a, b in ARB_TRIPLES])
def test_arbitrary_stream_device_equals_host(tx, th):
    rng = np.random.default_rng(31)
    rate = 0.98
    h = dsp.resample_filter(rate, 32).astype(th)
    nch = 3
    tol = 2e-6 if np.dtype(th) == F32 and np.dtype(tx) in (F32, C64) else 1e-11
    for aligned in (True, False):
        for sizes in ([8], [64, 4, 296, 5], None):      # 16-byte column strides except 5 and most random lengths
            x = rng.standard_normal((700, nch))
            if tx.kind == "c":
                x = x + 1j * rng.standard_normal((700, nch))
            x = x.astype(tx)
            f = dsp.FIRFilter(h, rate, 32, device=True)
            g = dsp.FIRFilter(h, rate, 32)
            ref = of.FIRArbitraryState(h, rate, 32)
            for t in (f, g, ref):
                t.setphase(0.3)
            buf, views = _arb_views(x, aligned, rng, sizes)
            for (a, b), xv in views:
                y = f.filt(xv).to_host()
                want = g.filt(x[a:b, 0])
                assert np.array_equal(y[:, 0], want), (aligned, sizes, a)
                lit = ref.filt(x[a:b, 0])
                assert lit.size == want.size
                if lit.size:
                    assert np.max(np.abs(want - lit)) <= tol * max(1.0, np.max(np.abs(lit))), (aligned, sizes, a)
                if f.history is not None:                 # None until the first non-empty chunk
                    assert np.array_equal(f.history.to_host()[:, 0], g.history)


@pytest.mark.gpu
def test_arbitrary_stream_banks_in_global_memory():
    rng = np.random.default_rng(55)
    rate = 1 / 55.55
    f, g = dsp.FIRFilter(None, rate, 32, device=True), dsp.FIRFilter(None, rate, 32)
    assert 2 * f.h.size * 8 > 96 * 1024 and f.h.dtype == np.float64
    ref = of.FIRArbitraryState(f.h, rate, 32)
    x = rng.standard_normal((4 * 3001, 2))
    total = 0
    for a in range(0, x.shape[0], 3001):
        y = f.filt(_dev_matrix(x[a:a + 3001])).to_host()
        want = g.filt(x[a:a + 3001, 1])
        lit = ref.filt(x[a:a + 3001, 1])
        assert np.array_equal(y[:, 1], want)
        assert np.max(np.abs(want - lit), initial=0.0) <= 1e-11 * max(1.0, np.max(np.abs(lit), initial=0.0))
        total += y.shape[0]
    assert total > 150


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [Fraction(3, 2), 0.98])
def test_launch_counts(ratio):
    rng = np.random.default_rng(9)
    h = dsp.resample_filter(ratio if isinstance(ratio, float) else ratio)
    h = h.astype(np.float32)
    f = dsp.FIRFilter(h, ratio, 32, device=True) if isinstance(ratio, float) else dsp.FIRFilter(h, ratio, device=True)
    x = rng.standard_normal((5000, 4)).astype(np.float32)
    chunks = [_dev_matrix(x[a:b]) for a, b in ((0, 1000), (1000, 1000), (1000, 1001), (1001, 5000))]
    dsp.filt(f, chunks[0])                                   # plan creation and first use outside the count
    f.setphase(9.0)
    for xd, limit in ((chunks[1], 0), (chunks[2], 1), (chunks[3], 2)):
        l0 = dsp.launch_count()
        y = dsp.filt(f, xd)
        used = dsp.launch_count() - l0
        assert used <= limit and (used >= 1 or xd.shape[0] == 0), (xd.shape, used)
        assert (y.shape[0] == 0) == (limit < 2)
    l0 = dsp.launch_count()
    for bad in (_dev_matrix(x[:10, :3]), DeviceArray((10, 4), np.float64)):
        with pytest.raises(dsp.ArgumentError):
            dsp.filt(f, bad)
    with pytest.raises(dsp.ArgumentError):
        dsp.filt_(chunks[3], f, chunks[3])
    assert dsp.launch_count() == l0


@pytest.mark.gpu
def test_c_abi_refuses_overlaps_before_any_launch():
    h = np.arange(1.0, 39.0, dtype=np.float32)
    plan = _lib.ResamplePlan(F32, h, 3, 2)
    arb = _lib.ResampleArbPlan(F32, h, 32)
    nx, nch, nout = 100, 2, 150                  # histories: 12 x 2 (rational plan), 1 x 2 (arbitrary plan)
    pool = DeviceArray((4096,), F32)
    p = pool.ptr
    xs, hi, ho, out = p, p + 4 * 1000, p + 4 * 1200, p + 4 * 1400
    bad = [(hi, hi + 4, xs, out, nout),          # hist_out overlaps hist_in
           (hi, xs + 16, xs, out, nout),         # hist_out overlaps x
           (hi, out + 4, xs, out, nout),         # hist_out overlaps out
           (hi, ho, xs, xs + 40, nout),          # out overlaps x
           (hi, ho, xs, hi - 4, nout),           # out overlaps hist_in
           (hi, ho, xs, out, nout + 1)]          # ldo < nout (ldo = nout below)
    l0 = dsp.launch_count()
    for hin, hout, x, o, n in bad:
        with pytest.raises(_lib.DSPB200Error) as e:
            plan.stream_exec_dev(hin, hout, x, nx, nch, 1, 0, o, nout, n, 0)
        assert e.value.code == _lib.EINVALID
        with pytest.raises(_lib.DSPB200Error) as e:
            arb.stream_exec_dev(hin, hout, x, nx, nch, 1, 0.0, 32 / 0.98, o, nout, n, 0)
        assert e.value.code == _lib.EINVALID
    with pytest.raises(_lib.DSPB200Error):                   # an empty chunk completes no output
        plan.stream_exec_dev(hi, ho, xs, 0, nch, 1, 0, out, nout, 3, 0)
    plan.stream_exec_dev(hi, ho, xs, 0, nch, 1, 0, out, nout, 0, 0)      # nx == 0: nothing to do
    assert dsp.launch_count() == l0
    plan.close()
    arb.close()
