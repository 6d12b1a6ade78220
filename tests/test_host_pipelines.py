"""Chunked host-pointer pipelines against their chunk schedules issued by hand.

`dspb200_welch_exec`, the long-column `dspb200_os_exec` and `dspb200_filt_welch_exec` stream the caller's buffer through
two device slots (`run_chunked`, csrc/runtime.cu).  Each must give, bit for bit and in as many kernel launches, what the
same device-pointer calls give when issued one by one from Python, every chunk copied into a buffer of its own.  The
chunk schedules are restated below from csrc/spectral.cu and csrc/overlap_save.cu.  A second call on the same plans must
repeat the first one's bits."""
import numpy as np
import pytest

from dspb200 import _lib
from dspb200.device import DeviceArray, to_device

pytestmark = pytest.mark.gpu

F32, F64, C64, C128 = (np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))
DTYPES = [F32, F64, C64, C128]
UINT = {4: np.uint32, 8: np.uint64, 16: np.uint64}
CHUNK_BYTES = 32 << 20


def _real(dt):
    return F64 if dt in (F64, C128) else F32


def _signal(rng, n, dt):
    part = np.float64 if dt in (F64, C128) else np.float32
    x = rng.standard_normal(n, dtype=part)
    if dt.kind == "c":
        x = x + 1j * rng.standard_normal(n, dtype=part)
    return np.ascontiguousarray(x.astype(dt))


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(UINT[a.dtype.itemsize]),
                                                                        b.view(UINT[b.dtype.itemsize]))


def _counted(fn):
    """(fn()'s result, the kernel launches it made)."""
    before = _lib.launch_count()
    res = fn()
    return res, _lib.launch_count() - before


# =============================================================================== chunk schedules

def welch_chunk_segs(itemsize, hop, k):
    """Segments per chunk of dspb200_welch_exec: about 32 MiB of new samples, at least 64."""
    return min(max((CHUNK_BYTES // itemsize) // hop, 64), k)


def os_chunk_out(itemsize, L):
    """Outputs per chunk of the long-column dspb200_os_exec: about 32 MiB, whole blocks; it streams nout > 2 chunks."""
    return ((CHUNK_BYTES // itemsize) // L + 1) * L


def filt_chunk(itemsize, L, n):
    """New samples per chunk of dspb200_filt_welch_exec: about 32 MiB, whole overlap-save blocks."""
    return min(max((CHUNK_BYTES // itemsize) // L * L, L), n)


# =============================================================================== hand-issued schedules

def _hand_welch(plan, x, r):
    k, hop = plan.nsegments(x.size), plan.n - plan.noverlap
    segs = welch_chunk_segs(x.itemsize, hop, k)
    out = DeviceArray((plan.nout,), _real(x.dtype))
    keep = []

    def run():
        plan.welch_begin_dev()
        for b0 in range(0, k, segs):
            b1 = min(b0 + segs, k)
            first, cnt = b0 * hop, (b1 - 1 - b0) * hop + plan.n
            keep.append(to_device(x[first:first + cnt]))
            plan.welch_accumulate_dev(keep[-1].ptr, cnt, first, b0, b1)
        plan.welch_finalize_dev(r, out.ptr)

    _, launches = _counted(run)
    return out.to_host(), launches


def _hand_os(plan, u, nout):
    nu, nv = u.size, plan.nv
    co = os_chunk_out(u.itemsize, plan.nfft - nv + 1)
    if nout <= 2 * co:                                     # staged: one device call over the whole column
        d, o = to_device(u), DeviceArray((nout,), u.dtype)
        _, launches = _counted(lambda: plan.exec_dev(d.ptr, nu, 1, o.ptr, nout))
        return o.to_host(), launches
    chunks = []

    def run():
        for m0 in range(0, nout, co):
            cnt = min(co, nout - m0)
            i_lo = max(m0 - (nv - 1), 0)
            ni = max(min(m0 + cnt, nu) - i_lo, 0)
            d = to_device(u[i_lo:i_lo + ni]) if ni else None
            o = DeviceArray((cnt,), u.dtype)
            plan.exec_range_dev(None if d is None else d.ptr, i_lo, ni, o.ptr, m0, cnt)
            chunks.append((m0, o, d))

    _, launches = _counted(run)
    out = np.concatenate([o.to_host() for _, o, _ in chunks])
    out[nu + nv - 1:] = 0                                  # the host call's outputs past the convolution are exact zeros
    return out, launches


def _hand_filt_welch(os_plan, plan, x, r):
    n, esz, halo = x.size, x.itemsize, os_plan.nv - 1
    k = plan.nsegments(n)
    chunk = filt_chunk(esz, os_plan.nfft - os_plan.nv + 1, n)
    out = DeviceArray((plan.nout,), _real(x.dtype))
    y = DeviceArray((n,), x.dtype)
    keep = []

    def run():
        plan.welch_begin_dev()
        done = 0
        for c0 in range(0, n, chunk) if k else ():
            c1 = min(c0 + chunk, n)
            in0 = max(c0 - halo, 0)
            keep.append(to_device(x[in0:c1]))
            os_plan.exec_range_dev(keep[-1].ptr, in0, c1 - in0, y.ptr + c0 * esz, c0, c1 - c0)
            hi = plan.nsegments(c1)
            if hi > done:
                plan.welch_accumulate_dev(y.ptr, c1, 0, done, hi)
                done = hi
        plan.welch_finalize_dev(r, out.ptr)

    _, launches = _counted(run)
    return out.to_host(), launches


# =============================================================================== host calls

def _host_welch(plan, x, r):
    out = np.full(plan.nout, np.nan, dtype=_real(x.dtype))
    _, launches = _counted(lambda: plan.welch(x, r, out))
    return out, launches


def _host_os(plan, u, nout):
    out = np.full(nout, np.nan, dtype=u.dtype)
    _, launches = _counted(lambda: plan.exec(u, out, u.size, 1, nout))
    return out, launches


def _host_filt_welch(os_plan, plan, x, r):
    out = np.full(plan.nout, np.nan, dtype=_real(x.dtype))
    _, launches = _counted(lambda: plan.filt_welch_ptr(os_plan, _lib.ptr(x) if x.size else None, x.size, r, _lib.ptr(out)))
    return out, launches


# =============================================================================== tests

@pytest.mark.parametrize("nfft", [4096, 1000], ids=["fused", "cufft"])
@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: d.name)
def test_welch_exec_matches_hand_schedule(dt, nfft):
    rng = np.random.default_rng([nfft, dt.num])
    hop = nfft // 2
    plan = _lib.SpecPlan(dt, nfft, nfft - hop, nfft, dt.kind != "c", np.hanning(nfft))
    try:
        chunk = welch_chunk_segs(dt.itemsize, hop, 1 << 40)
        for k in (1, chunk, chunk + 1, 2 * chunk + 9):
            x = _signal(rng, (k - 1) * hop + nfft + hop // 3, dt)   # a tail that completes no segment
            assert plan.nsegments(x.size) == k
            r = 0.375 * k
            host, n_host = _host_welch(plan, x, r)
            ref, n_ref = _hand_welch(plan, x, r)
            assert _same(host, ref), k
            assert n_host == n_ref, k
            assert _same(_host_welch(plan, x, r)[0], host), k
    finally:
        plan.close()


def _os_cases(esz, L, nv):
    """(nu, nout): the staged limit nout = 2 chunks, one block past it, and an odd count past it, each with nout = nu and
    nout = nu + nv - 1; then nout past nu + nv - 1, so that the last chunk reads no input."""
    co = os_chunk_out(esz, L)
    return [(nout - d, nout) for nout in (2 * co, 2 * co + L, 2 * co + L // 2 + 7) for d in (0, nv - 1)] + [(co, 2 * co + L)]


@pytest.mark.parametrize("dt,nv,nfft", [(F32, 1025, 0), (C128, 513, 0), (C64, 301, 3000)],
                         ids=["f32-fused", "c128-fused", "c64-cufft"])
def test_os_exec_long_column_matches_hand_schedule(dt, nv, nfft):
    rng = np.random.default_rng([nv, dt.num])
    plan = _lib.OsPlan(_signal(rng, nv, dt), nfft)
    try:
        assert plan.fused == (nfft == 0)
        L = plan.nfft - nv + 1
        for nu, nout in _os_cases(dt.itemsize, L, nv):
            u = _signal(rng, nu, dt)
            host, n_host = _host_os(plan, u, nout)
            ref, n_ref = _hand_os(plan, u, nout)
            assert _same(host, ref), (nu, nout)
            assert n_host == n_ref, (nu, nout)
            if nout > nu + nv - 1:
                assert not np.any(host[nu + nv - 1:])
            assert _same(_host_os(plan, u, nout)[0], host), (nu, nout)
    finally:
        plan.close()


# the three cases of test_gpu_parity.py::test_filt_welch_pipeline_matches_the_two_calls
FILT_CASES = [(C64, (1 << 23) + 12345, 1025), (F32, 3_000_001, 257), (F64, 400_000, 129)]


def _filt_plans(rng, dt, nb):
    os_plan = _lib.OsPlan(_signal(rng, nb, dt), 0)
    plan = _lib.SpecPlan(dt, 4096, 2048, 4096, dt.kind != "c", np.hanning(4096))
    return os_plan, plan


def _check_filt_welch(os_plan, plan, x):
    r = 0.5 * max(plan.nsegments(x.size), 1)
    host, n_host = _host_filt_welch(os_plan, plan, x, r)
    ref, n_ref = _hand_filt_welch(os_plan, plan, x, r)
    assert _same(host, ref), x.size
    assert n_host == n_ref, x.size
    return host


@pytest.mark.parametrize("dt,n,nb", FILT_CASES, ids=lambda v: getattr(v, "name", str(v)))
def test_filt_welch_matches_hand_schedule(dt, n, nb):
    rng = np.random.default_rng([n, nb])
    os_plan, plan = _filt_plans(rng, dt, nb)
    try:
        x = _signal(rng, n, dt)
        first = _check_filt_welch(os_plan, plan, x)
        short = _signal(rng, n // 3, dt)                     # a different n on the same plans, then the first call again
        _check_filt_welch(os_plan, plan, short)
        assert _same(_host_filt_welch(os_plan, plan, x, 0.5 * plan.nsegments(n))[0], first)
    finally:
        os_plan.close()
        plan.close()


def test_filt_welch_one_chunk_and_no_segment():
    rng = np.random.default_rng(11)
    os_plan, plan = _filt_plans(rng, F32, 257)
    try:
        L = os_plan.nfft - os_plan.nv + 1
        n = filt_chunk(4, L, 1 << 40)                        # exactly one whole chunk
        assert filt_chunk(4, L, n) == n and n > 4096
        _check_filt_welch(os_plan, plan, _signal(rng, n, F32))
        for n in (4095, 0):                                  # k == 0: no chunk, the PSD of no segment
            assert plan.nsegments(n) == 0
            _check_filt_welch(os_plan, plan, _signal(rng, n, F32))
    finally:
        os_plan.close()
        plan.close()
