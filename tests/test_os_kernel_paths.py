"""Every overlap-save kernel instance and entry point (csrc/overlap_save.cu) exactly against an integer convolution.

A plan with a power-of-two nfft = N in 32 .. 16384 (Float32) or 32 .. 8192 (Float64) runs `os_fused_kernel<T, N, CPLX>`,
38 instances in all; each has an edge form and an interior form of its unit (`os_unit<..., INTERIOR>`).  Any other nfft
runs the cuFFT generic path.  The entry points are `exec_dev` (columns of a device matrix), `exec_range_dev` (a range of
outputs from a local slice of the input) and the host `exec`, which streams one long column in chunks.  The routing, the
per-unit geometry of the fused kernel, the generic path's batch and the host chunk are restated below, so that the case
table can show what it reaches.

The main check is exact.  Samples are integers in [-8, 8] and taps nonzero integers in [-4, 4] (both parts of complex
data), so the true convolution is an integer.  The FFT result is off by far less than 0.5 from it (a float32 pocketfft
overlap-save at N = 16384, 4097 .. 16384 taps, outputs up to 1.1e4: at most 0.003), so rint(y) must equal the integer
convolution bit for bit, whatever the kernel.  Besides, |y - exact| must stay within 2^-4 (Float32) or 1e-9 (Float64),
so that a subtle arithmetic defect still shows.  Outputs at or past nu + nv - 1 are exact zeros (src/dspbase.jl:733-735):
they must be bitwise +0, not merely round to 0.  Inputs sit between sentinel samples of magnitude 1000 and outputs between
NaN cells: the taps being nonzero, one read outside the stored range changes a rounded output, and one write outside
the output range leaves a NaN cell changed.

The reference is np.convolve on integers for small cases and rint(scipy.signal.oaconvolve) in float64 for large ones,
which must lie within 1e-3 of its rounding.  The CPU tests check the reference and the coverage of the case table; the
rest need a GPU."""
import math

import numpy as np
import pytest
from scipy import signal as ss

from conftest import relerr

F32, F64, C64, C128 = (np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))
SIZES = (32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384)          # DSP_OS_SIZES, overlap_save.cu:619
INSTANCES = [(dt, N) for dt in (F32, C64) for N in SIZES] + [(dt, N) for dt in (F64, C128) for N in SIZES if N <= 8192]
H100_SMS = 132
MAX_THREADS_PER_SM = 2048
GUARD = 64                # sentinel / NaN cells on each side of a device buffer


def _cplx(dt):
    return np.dtype(dt).kind == "c"


def _f64(dt):
    return np.dtype(dt) in (F64, C128)


def _inst_id(inst):
    dt, N = inst
    return f"{dt.name}-{N}"


# =============================================================================== routing restated from overlap_save.cu

def auto_nfft(nv, f64):
    """auto_nfft (overlap_save.cu:794-807): the cheapest power of two 1024 .. nmax that leaves at least half of every
    block new output, else the generic path's power of two >= 4 nv."""
    nmax = 8192 if f64 else 16384
    best, best_cost = 0, 0.0
    n = 1024
    while n <= nmax:
        if n - nv + 1 >= n // 2:
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
    """os_fused_ok (overlap_save.cu:621-625)."""
    return 32 <= nfft <= (8192 if f64 else 16384) and nfft & (nfft - 1) == 0 and nfft >= nv


def fft_threads(N):
    """fft_threads (fft_core.cuh:667-670)."""
    nb16 = N // 16
    return 64 if nb16 < 64 else (512 if nb16 > 512 else (256 if nb16 > 256 else nb16))


def os_threads(N, f64, cplx):
    """os_threads (overlap_save.cu:83-91): (threads per CTA, wide: 1024 resident threads, staged: TMA-staged input)."""
    f32 = not f64
    wide = f32 and (512 <= N <= 4096 or (N == 256 and not cplx))
    return fft_threads(N), wide, f32 and N == 16384


def resident_bound(N):
    """Upper bound on the resident CTAs of a fused launch: 132 SMs, 2048 threads each."""
    return H100_SMS * MAX_THREADS_PER_SM // fft_threads(N)


def generic_batch(nfft):
    """Blocks per cuFFT batch of the generic path (overlap_save.cu:1035-1037)."""
    return min(max((1 << 22) // nfft, 1), 4096)


def chunk_out(itemsize, L):
    """Outputs per chunk of the host path (overlap_save.cu:1127): about 32 MiB, whole blocks."""
    return ((32 << 20) // itemsize // L + 1) * L


def host_chunked(ncols, nu, nout, itemsize, L):
    """Whether the host exec streams the call in chunks (overlap_save.cu:1128)."""
    return ncols == 1 and nout > 2 * chunk_out(itemsize, L) and nu > 0


def _clamp(v):
    return max(-(1 << 30), min(1 << 30, v))


def unit_geometry(dt, N, nv, *, nu_local, out_count, u_begin=0, out_begin=0, zero_from=None, ncols=1, u_col_stride=0,
                  u_offset=0):
    """Per unit of one fused launch, in launch order: the `geometry` and `stage_src` lambdas of os_fused_kernel
    (overlap_save.cu:337-376).  zero_from None is the range form's "no limit"; u_offset is the input's offset in elements
    from a 16-byte aligned address.  Each unit is a dict: col, interior, staged, starts_before (jlo > 0, the unit begins
    before the stored signal), forced_zeros (jzero < span), b_past_end (real: block B wants no output)."""
    cplx, f64 = _cplx(dt), _f64(dt)
    esz = np.dtype(dt).itemsize
    L = N - nv + 1
    span = N if cplx else N + L
    stage_bytes = (span * esz + 15) & ~15
    staged_kernel = os_threads(N, f64, cplx)[2]
    nblk = -(-out_count // L)
    upc = nblk if cplx else (nblk + 1) // 2
    units = []
    for gu in range(upc * ncols):
        col, unit = divmod(gu, upc)
        q = unit if cplx else 2 * unit
        s0 = out_begin + q * L - (nv - 1)
        i0 = s0 - u_begin
        jlo, jhi, jend = _clamp(-i0), _clamp(nu_local - i0), _clamp(out_begin + out_count - s0)
        jzero = (1 << 30) if zero_from is None else _clamp(zero_from - s0)
        interior = jlo <= 0 and jhi >= span and jend >= span and jzero >= span
        aligned = (u_offset + col * u_col_stride + i0) * esz % 16 == 0
        units.append(dict(col=col, interior=interior, staged=staged_kernel and interior and jhi * esz >= stage_bytes and aligned,
                          starts_before=jlo > 0, forced_zeros=jzero < span, b_past_end=not cplx and jend <= N))
    return units


# =============================================================================== reference

def int_taps(rng, nv, dt):
    """Nonzero integer taps in [-4, 4] (both parts for complex)."""
    def part():
        return rng.choice(np.array([-4, -3, -2, -1, 1, 2, 3, 4]), nv).astype(np.float64)
    v = part() + 1j * part() if _cplx(dt) else part()
    return v.astype(dt)


def int_signal(rng, shape, dt):
    v = rng.integers(-8, 9, shape).astype(np.float64)
    if _cplx(dt):
        v = v + 1j * rng.integers(-8, 9, shape)
    return v.astype(dt)


def _exact_1d(u, v, direct_limit=4_000_000):
    cplx = _cplx(u.dtype) or _cplx(v.dtype)
    if u.size * v.size <= direct_limit:
        def c(a, b):
            return np.convolve(np.rint(a).astype(np.int64), np.rint(b).astype(np.int64)).astype(np.float64)
        if not cplx:
            return c(u, v)
        return (c(u.real, v.real) - c(u.imag, v.imag)) + 1j * (c(u.real, v.imag) + c(u.imag, v.real))
    f = ss.oaconvolve(u.astype(np.complex128 if cplx else np.float64), v.astype(np.complex128 if cplx else np.float64))
    r = np.rint(f.real) + 1j * np.rint(f.imag) if cplx else np.rint(f)
    assert np.abs(f - r).max() <= 1e-3
    return r


def exact_conv(u, v, nout=None, direct_limit=4_000_000):
    """Full convolution of the integer-valued columns of u ((nu,) or (nu, ncols)) with v, float64 / complex128 holding
    exact integers; cut or zero-padded to nout samples."""
    u2 = u.reshape(u.shape[0], -1)
    full = u2.shape[0] + v.size - 1
    nout = full if nout is None else nout
    cplx = _cplx(u.dtype) or _cplx(v.dtype)
    out = np.zeros((nout, u2.shape[1]), dtype=np.complex128 if cplx else np.float64)
    for c in range(u2.shape[1]):
        y = _exact_1d(u2[:, c], v, direct_limit)
        out[:min(nout, full), c] = y[:nout]
    return out.reshape(nout) if u.ndim == 1 else out


def check_exact(y, want, f64, zero_from=None, what=""):
    """rint(y) equals the integer convolution bit for bit, |y - exact| within 2^-4 (Float32) or 1e-9 (Float64), and rows
    from zero_from on are bitwise +0.  Returns max |y - exact|."""
    assert y.shape == want.shape, what
    yr = y.astype(np.complex128)
    ok = (np.rint(yr.real) == want.real) & (np.rint(yr.imag) == np.asarray(want).imag)
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, (what, bad.size, bad[:8])
    err = float(np.abs(yr - want).max()) if y.size else 0.0
    assert err <= (1e-9 if f64 else 2.0 ** -4), (what, err)
    if zero_from is not None and zero_from < y.shape[0]:
        tail = np.ascontiguousarray(y[zero_from:])
        bits = tail.view(np.uint32 if tail.dtype in (F32, C64) else np.uint64)
        assert not bits.any(), (what, "forced zeros are not +0", np.flatnonzero(bits.reshape(tail.shape[0], -1).any(axis=1))[:8])
    return err


# =============================================================================== case tables

def dev_cases(dt, N):
    """(nv, nu, nout) of test_every_instance_exact_with_guards: nv in {1, 2, N/2+1, N-1, N} (L = N .. 1), nu in {1, < nv,
    L-1, L, L+1, many blocks}, nout in {nu (fftfilt), nu+nv-1 (conv), nu+nv-1+2L+3 (forced zeros)}.  With nv = N the many
    blocks outnumber the resident CTAs, so persistent CTAs loop."""
    cplx = _cplx(dt)
    per = 1 if cplx else 2
    cases = []
    for nv in sorted({1, 2, N // 2 + 1, N - 1, N}):
        L = N - nv + 1
        span = N if cplx else N + L
        many = (nv - 1) + 2 * span + 3 * L + 3
        if nv == N:
            many = max(many, per * resident_bound(N) + 2 * span + 3)
        for nu in sorted({1, nv - 1, L - 1, L, L + 1, many} - {0}):
            for nout in sorted({nu, nu + nv - 1, nu + nv - 1 + 2 * L + 3}):
                cases.append((nv, nu, nout))
    return cases


def column_case(dt, N):
    """(nv, nu) of the column tests: nv = N/4 + 1 (4097 taps at N = 16384: the staged kernels), an odd block count per
    column and an odd nu, so that columns start at differently aligned addresses.  101 blocks: even three real columns
    hold more units than the staged kernels have CTAs (one per SM), so CTAs go on to units of later columns."""
    nv = N // 4 + 1
    L = N - nv + 1
    nu = 100 * L + L // 2 + 1 - (nv - 1)
    return nv, nu


def range_case(N):
    """(nv, nu, ranges) of test_exec_range_dev_exact: ranges (out_begin, out_count) off the block grid, shorter than a
    block, from u_begin > 0 on, across the end of the output and wholly past it."""
    nv = N // 2 + 1
    L = N - nv + 1
    nu = 5 * L + 3
    full = nu + nv - 1
    return nv, nu, [(0, full), (0, 1), (1, L - 1), (L + 3, 2 * L + 5), (nv + 6, 3 * L), (nv - 1, L),
                    (full - 2, L + 5), (full + 4, L + 2), (full + 3 * L, 3)]


def host_cases():
    """(dtype, nfft, nv, nout) of test_host_exec_chunked: just above the chunking threshold, one chunk block count odd and
    one even per type."""
    cases = []
    for dt, nfft in ((F32, 4096), (F64, 2048), (C128, 1024)):
        found = {}
        for nv in range(301, nfft):
            L = nfft - nv + 1
            k = chunk_out(dt.itemsize, L) // L
            found.setdefault(k % 2, nv)
            if len(found) == 2:
                break
        for parity in (1, 0):
            nv = found[parity]
            L = nfft - nv + 1
            cases.append((dt, nfft, nv, 2 * chunk_out(dt.itemsize, L) + L // 2 + 7))
    return cases


# (dtype, nfft, nv, ncols, nblk): the generic path, several batches with a partial last one
GENERIC_CASES = [(F32, 1000, 37, 2, generic_batch(1000) + 3), (C64, 3000, 1001, 2, generic_batch(3000) + 3),
                 (F32, 32768, 5000, 1, 2 * generic_batch(32768) + 3), (F32, 65536, 40001, 1, generic_batch(65536) + 3),
                 (F64, 16384, 3000, 2, generic_batch(16384) + 3), (C128, 16384, 16384, 1, 64 * generic_batch(16384) + 24)]


def _generic_nu(nfft, nv, nblk):
    """nu whose forced-zero call (nout = nu + nv - 1 + 2L + 3) has nblk blocks, the last one partial."""
    L = nfft - nv + 1
    return max(1, (nblk - 1) * L + L // 2 + 1 - (nv - 1) - 2 * L - 3)


# =============================================================================== CPU: the reference and the table

def test_reference_matches_direct_convolution():
    rng = np.random.default_rng(1)
    for dt in (F64, C128):
        for nu, nv, ncols in ((1, 1, 1), (7, 13, 2), (300, 41, 3), (2000, 999, 1)):
            u = int_signal(rng, (nu, ncols), dt)
            v = int_taps(rng, nv, dt)
            direct = exact_conv(u, v)
            via_fft = exact_conv(u, v, direct_limit=0)
            assert np.array_equal(direct, via_fft), (dt, nu, nv)
            assert np.array_equal(direct[:, 0], np.convolve(u[:, 0].astype(np.complex128), v.astype(np.complex128)))
            assert np.array_equal(exact_conv(u, v, nu + nv + 4)[nu + nv - 1:], np.zeros((5, ncols)))
    assert np.all(int_taps(rng, 1000, F32) != 0) and np.all(int_taps(rng, 1000, C64).real != 0)


def test_restated_routing():
    # auto_nfft: the cost model's picks (513 taps: 4096 and 8192 cost the same, the smaller wins), the half-new-output
    # limit, then the generic fallback
    assert [auto_nfft(nv, False) for nv in (1, 64, 513, 2049, 4097, 8193, 8194, 9000)] == \
        [1024, 1024, 4096, 16384, 16384, 16384, 65536, 65536]
    assert auto_nfft(2049, True) == 8192 and auto_nfft(4097, True) == 8192 and auto_nfft(4098, True) == 32768
    assert os_fused_ok(16384, 16384, False) and not os_fused_ok(16384, 1, True) and not os_fused_ok(1000, 3, False)
    assert not os_fused_ok(16, 3, False) and not os_fused_ok(32, 33, False)
    assert [fft_threads(N) for N in SIZES] == [64, 64, 64, 64, 64, 64, 128, 256, 256, 512]
    assert [N for N in SIZES if os_threads(N, False, True)[1]] == [512, 1024, 2048, 4096]
    assert [N for N in SIZES if os_threads(N, False, False)[1]] == [256, 512, 1024, 2048, 4096]
    assert [(N, f64) for N in SIZES for f64 in (False, True) if os_threads(N, f64, True)[2]] == [(16384, False)]
    assert generic_batch(1000) == 4096 and generic_batch(3000) == 1398 and generic_batch(65536) == 64
    assert chunk_out(4, 4096) == 2049 * 4096 and chunk_out(16, 1) == (1 << 21) + 1


def test_case_table_covers_every_kernel_family():
    assert len(INSTANCES) == 38
    for dt, N in INSTANCES:
        cplx, f64 = _cplx(dt), _f64(dt)
        seen = dict(starts_before=False, interior=False, tail=False, forced_zeros=False, b_past_end=False, loops=False)
        for nv, nu, nout in dev_cases(dt, N):
            assert os_fused_ok(N, nv, f64)
            units = unit_geometry(dt, N, nv, nu_local=nu, out_count=nout, zero_from=nu + nv - 1)
            seen["starts_before"] |= any(u["starts_before"] for u in units)
            seen["interior"] |= any(u["interior"] for u in units)
            seen["tail"] |= any(not u["interior"] and not u["starts_before"] for u in units)
            seen["forced_zeros"] |= any(u["forced_zeros"] for u in units)
            seen["b_past_end"] |= any(u["b_past_end"] for u in units)        # real: odd block count
            seen["loops"] |= len(units) > resident_bound(N)
        if cplx:
            seen["b_past_end"] = True
        assert all(seen.values()), (dt, N, seen)
        # the column case: an odd block count per column; its interior units start at differently aligned addresses
        nv, nu = column_case(dt, N)
        L = N - nv + 1
        assert -(-(nu + nv - 1) // L) % 2 == 1 and nu % 2 == 1
        # the range case reaches the edge and the interior form from u_begin > 0, out_begin off the block grid
        nv, nu, ranges = range_case(N)
        assert any(b % (N - nv + 1) != 0 and b >= nv - 1 for b, _ in ranges)
        assert any(c < N - nv + 1 for _, c in ranges) and any(b > nu + nv - 1 for b, _ in ranges)
    # both TMA-staged kernels: staged and unstaged interior units inside one multi-column launch, and CTAs whose next
    # unit lies in the next column
    for dt in (F32, C64):
        nv, nu = column_case(dt, 16384)
        assert nv == 4097
        for ncols in (3, 5):
            units = unit_geometry(dt, 16384, nv, nu_local=nu, out_count=nu + nv - 1, zero_from=nu + nv - 1, ncols=ncols,
                                  u_col_stride=nu)
            assert {u["staged"] for u in units if u["interior"]} == {True, False}
            assert len({u["col"] for u in units if u["staged"]}) < ncols
            nxt = [(a, b) for a, b in zip(units, units[H100_SMS:]) if a["col"] != b["col"]]
            assert any(a["interior"] and b["interior"] for a, b in nxt)
    # the host path streams Float32, Float64 and ComplexF64 columns in chunks of an odd and an even block count
    hc = host_cases()
    for dt in (F32, F64, C128):
        parities = set()
        for cdt, nfft, nv, nout in hc:
            if cdt == dt:
                L = nfft - nv + 1
                assert os_fused_ok(nfft, nv, _f64(dt))
                assert host_chunked(1, nout - nv + 1, nout, dt.itemsize, L)
                assert nout < 2 * chunk_out(dt.itemsize, L) + L                     # just above the threshold
                parities.add(chunk_out(dt.itemsize, L) // L % 2)
        assert parities == {0, 1}, dt
    # the generic path: non-power-of-two sizes and sizes above the fused limit, several batches, a partial last one
    for dt, nfft, nv, ncols, nblk in GENERIC_CASES:
        assert not os_fused_ok(nfft, nv, _f64(dt))
        L = nfft - nv + 1
        nu = _generic_nu(nfft, nv, nblk)
        assert -(-(nu + nv - 1 + 2 * L + 3) // L) == nblk
        assert nblk > generic_batch(nfft) and nblk % generic_batch(nfft) != 0
    assert {n for _, n, _, _, _ in GENERIC_CASES} >= {1000, 3000, 32768, 65536, 16384}
    assert any(c > 1 for *_, c, _ in GENERIC_CASES)


# =============================================================================== GPU helpers

@pytest.fixture(scope="module")
def dsp():
    return pytest.importorskip("dspb200")


def _sentinels(rng, n, dt):
    s = rng.choice(np.array([-1000.0, 1000.0]), n)
    if _cplx(dt):
        s = s + 1j * rng.choice(np.array([-1000.0, 1000.0]), n)
    return s.astype(dt)


class Guarded:
    """A device buffer of GUARD cells, `n` data cells (from `offset` cells on) and GUARD cells: sentinels (input) or NaN
    (output) outside the data."""

    def __init__(self, dt, n, rng=None, data=None, offset=0):
        from dspb200 import device
        self.dt, self.n, self.lo = np.dtype(dt), n, GUARD + offset
        if rng is None:
            host = np.full(self.lo + n + GUARD, np.nan, dtype=dt)
        else:
            host = _sentinels(rng, self.lo + n + GUARD, dt)
        if data is not None:
            host[self.lo:self.lo + n] = np.asarray(data).ravel(order="F")
        self.host = host
        self.buf = device.to_device(host)
        self.ptr = self.buf.ptr + self.lo * self.dt.itemsize

    def data(self, shape=None):
        """The data cells (Fortran-ordered `shape`), after checking that the cells around them are unchanged."""
        h = self.buf.to_host()
        outside = np.concatenate([h[:self.lo], h[self.lo + self.n:]])
        want = np.concatenate([self.host[:self.lo], self.host[self.lo + self.n:]])
        assert np.array_equal(outside, want, equal_nan=True), "a cell outside the buffer's range changed"
        d = h[self.lo:self.lo + self.n]
        return d if shape is None else d.reshape(shape, order="F")


def _exec_dev(dsp, plan, u, nout, offset=0, rng=None):
    """plan.exec_dev on u ((nu,) or (nu, ncols)) inside a guarded buffer; one launch for a fused plan.  Returns y."""
    from dspb200 import device
    rng = rng if rng is not None else np.random.default_rng(0)
    ncols = 1 if u.ndim == 1 else u.shape[1]
    nu = u.shape[0]
    gu = Guarded(u.dtype, u.size, rng=rng, data=u, offset=offset)
    go = Guarded(u.dtype, nout * ncols)
    n0 = dsp.launch_count()
    plan.exec_dev(gu.ptr, nu, ncols, go.ptr, nout, 0)
    device.sync()
    if plan.fused:
        assert dsp.launch_count() - n0 == 1
    gu.data()
    return go.data((nout, ncols) if u.ndim == 2 else (nout,))


def _plan(dsp, v, nfft):
    plan = dsp._lib.OsPlan(v, nfft)
    assert plan.nfft == (nfft or auto_nfft(v.size, _f64(v.dtype)))
    assert plan.fused == os_fused_ok(plan.nfft, v.size, _f64(v.dtype))
    return plan


def _report(what, err):
    print(f"max|y - exact| {what}: {err:.3g}")


# =============================================================================== GPU: the fused instances

@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", INSTANCES, ids=[_inst_id(i) for i in INSTANCES])
def test_every_instance_exact_with_guards(dsp, dt, N):
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num])
    f64 = _f64(dt)
    worst = 0.0
    plans = {}
    try:
        for nv, nu, nout in dev_cases(dt, N):
            if nv not in plans:
                v = int_taps(rng, nv, dt)
                plans[nv] = (_plan(dsp, v, N), v)
                assert plans[nv][0].fused
            plan, v = plans[nv]
            u = int_signal(rng, nu, dt)
            y = _exec_dev(dsp, plan, u, nout, rng=rng)
            worst = max(worst, check_exact(y, exact_conv(u, v, nout), f64, nu + nv - 1, (nv, nu, nout)))
    finally:
        for p, _ in plans.values():
            p.close()
        device.empty_cache()
    _report(_inst_id((dt, N)), worst)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", INSTANCES, ids=[_inst_id(i) for i in INSTANCES])
def test_columns_exact(dsp, dt, N):
    # distinct data per column and an odd block count per column, so that a leak between columns or a wrong pairing of
    # the last real block shows; at N = 16384 (4097 taps) staged and unstaged units alternate between the columns
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 3])
    nv, nu = column_case(dt, N)
    v = int_taps(rng, nv, dt)
    plan = _plan(dsp, v, N)
    try:
        for ncols in (3, 5):
            u = int_signal(rng, (nu, ncols), dt)
            nout = nu + nv - 1
            y = _exec_dev(dsp, plan, u, nout, rng=rng)
            check_exact(y, exact_conv(u, v), _f64(dt), nout, ncols)
            y = _exec_dev(dsp, plan, u, nu + 3, offset=1, rng=rng)               # fftfilt length, shifted alignment
            check_exact(y, exact_conv(u, v, nu + 3), _f64(dt), nout, ncols)
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F64])
def test_fftfilt_matrix_host_and_device_exact(dsp, dt):
    from dspb200 import device
    rng = np.random.default_rng([dt.num, 5])
    for nfft, nv, nx, ncols in ((1024, 300, 7 * 725 + 11, 3), (4096, 1000, 5 * 3097 + 2, 5)):
        b = int_taps(rng, nv, dt)
        x = np.asfortranarray(int_signal(rng, (nx, ncols), dt))
        want = exact_conv(x, b, nx)
        check_exact(dsp.fftfilt(b, x, nfft), want, _f64(dt), what=("host", nfft))
        y = dsp.fftfilt(b, device.to_device(x), nfft)
        check_exact(y.to_host(), want, _f64(dt), what=("device", nfft))
    device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", INSTANCES, ids=[_inst_id(i) for i in INSTANCES])
def test_exec_range_dev_exact(dsp, dt, N):
    # each range gets exactly the input samples it reads, between sentinels, at their global offset
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 7])
    nv, nu, ranges = range_case(N)
    v = int_taps(rng, nv, dt)
    u = int_signal(rng, nu, dt)
    plan = _plan(dsp, v, N)
    try:
        full = exact_conv(u, v, nu + nv - 1 + 4 * N)
        for b, c in ranges:
            lo = min(nu, max(0, b - (nv - 1)))
            hi = max(lo, min(nu, b + c))
            gu = Guarded(dt, hi - lo, rng=rng, data=u[lo:hi])
            go = Guarded(dt, c)
            n0 = dsp.launch_count()
            plan.exec_range_dev(gu.ptr, lo, hi - lo, go.ptr, b, c, 0)
            device.sync()
            assert dsp.launch_count() - n0 == 1
            gu.data()
            check_exact(go.data(), full[b:b + c], _f64(dt), what=(b, c))
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
def test_auto_nfft_matches_restatement(dsp):
    rng = np.random.default_rng(9)
    for dt in (F32, F64, C64, C128):
        for nv in (1, 2, 100, 257, 513, 514, 1000, 1025, 2049, 2050, 4097, 4098, 8193, 8194):
            plan = _plan(dsp, int_taps(rng, nv, dt), 0)
            plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", INSTANCES, ids=[_inst_id(i) for i in INSTANCES])
def test_precision_random_data_per_block(dsp, dt, N):
    # Gaussian data against the float64 convolution, measured over each block of L outputs
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 11])
    cplx = _cplx(dt)
    nv = N // 2 + 1
    L = N - nv + 1
    nu = 9 * L + 5

    def gauss(n):
        g = rng.standard_normal(n)
        return (g + 1j * rng.standard_normal(n) if cplx else g).astype(dt)
    u, v = gauss(nu), gauss(nv)
    plan = _plan(dsp, v, N)
    try:
        y = _exec_dev(dsp, plan, u, nu + nv - 1, rng=rng)
    finally:
        plan.close()
        device.empty_cache()
    w = np.complex128 if cplx else np.float64
    truth = np.convolve(u.astype(w), v.astype(w))
    nb = -(-truth.size // L)
    errs = np.array([relerr(y[k * L:(k + 1) * L], truth[k * L:(k + 1) * L]) for k in range(nb)])
    # (a block with an unwritten, NaN output has a NaN error, which must fail: no max() that skips it)
    assert np.all(errs < (1e-12 if _f64(dt) else 1e-6)), errs
    print(f"largest per-block relative error {_inst_id((dt, N))}: {errs.max():.3g}")


# =============================================================================== GPU: the generic path

@pytest.mark.gpu
@pytest.mark.parametrize("dt,nfft,nv,ncols,nblk", GENERIC_CASES,
                         ids=[f"{c[0].name}-{c[1]}-nv{c[2]}-c{c[3]}" for c in GENERIC_CASES])
def test_generic_path_exact(dsp, dt, nfft, nv, ncols, nblk):
    from dspb200 import device
    rng = np.random.default_rng([nfft, nv, dt.num])
    L = nfft - nv + 1
    nu = _generic_nu(nfft, nv, nblk)
    v = int_taps(rng, nv, dt)
    plan = _plan(dsp, v, nfft)
    assert not plan.fused
    try:
        u = int_signal(rng, (nu, ncols), dt)
        nout = nu + nv - 1 + 2 * L + 3
        n0 = dsp.launch_count()
        y = _exec_dev(dsp, plan, u, nout, rng=rng)
        # per column and batch: gather, forward transform, product, inverse transform, scatter
        assert dsp.launch_count() - n0 == 5 * ncols * -(-nblk // generic_batch(nfft))
        want = exact_conv(u, v, nout + L + 16)
        _report(f"generic {dt.name} nfft {nfft}", check_exact(y, want[:nout], _f64(dt), nu + nv - 1, "exec_dev"))
        for b, c in ((3, L - 1), (L + 5, 3 * L + 2), (nu + nv - 3, L + 7)):
            lo = min(nu, max(0, b - (nv - 1)))
            hi = max(lo, min(nu, b + c))
            gu = Guarded(dt, hi - lo, rng=rng, data=u[lo:hi, 0])
            go = Guarded(dt, c)
            plan.exec_range_dev(gu.ptr, lo, hi - lo, go.ptr, b, c, 0)
            device.sync()
            gu.data()
            check_exact(go.data(), want[b:b + c, 0], _f64(dt), what=("range", b, c))
    finally:
        plan.close()
        device.empty_cache()


# =============================================================================== GPU: the host entry point

@pytest.mark.gpu
@pytest.mark.parametrize("dt,nfft,nv,nout", host_cases(),
                         ids=[f"{c[0].name}-nv{c[2]}-k{chunk_out(c[0].itemsize, c[1] - c[2] + 1) // (c[1] - c[2] + 1)}"
                              for c in host_cases()])
def test_host_exec_chunked(dsp, dt, nfft, nv, nout):
    # one long column streamed in chunks of whole blocks; a real chunk with an odd block count pairs its blocks
    # differently from one call, a complex one computes the very same blocks as exec_dev
    from dspb200 import device
    rng = np.random.default_rng([nfft, nv, dt.num])
    nu = nout - nv + 1
    v = int_taps(rng, nv, dt)
    u = int_signal(rng, nu, dt)
    plan = _plan(dsp, v, nfft)
    try:
        y = np.full(nout, np.nan, dtype=dt)
        plan.exec(u, y, nu, 1, nout)
        _report(f"host {dt.name} nv {nv}", check_exact(y, exact_conv(u, v), _f64(dt)))
        if _cplx(dt):
            assert np.array_equal(y, _exec_dev(dsp, plan, u, nout, rng=rng))
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F64, C64, C128])
def test_host_exec_columns(dsp, dt):
    from dspb200 import device
    rng = np.random.default_rng([dt.num, 13])
    for nfft, nv, nu, ncols in ((512, 129, 7 * 384 + 5, 3), (16384 if not _f64(dt) else 8192, 2000, 50_001, 2)):
        v = int_taps(rng, nv, dt)
        u = np.asfortranarray(int_signal(rng, (nu, ncols), dt))
        plan = _plan(dsp, v, nfft)
        try:
            for nout in (nu, nu + nv - 1, nu + nv + 40):
                y = np.full((nout, ncols), np.nan, dtype=dt, order="F")
                plan.exec(u, y, nu, ncols, nout)
                check_exact(y, exact_conv(u, v, nout), _f64(dt), nu + nv - 1, (nfft, nout))
        finally:
            plan.close()
    device.empty_cache()
