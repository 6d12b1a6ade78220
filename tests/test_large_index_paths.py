"""The entry points past 32-bit indices: range offsets far beyond 2^32 samples, and calls over 2^31 elements and 4 GiB.

Index arithmetic fails at two limits: element index 2^31, where an `int` overflows, and byte offset 2^32, where a
`uint32_t` byte count or offset does.  The kernels keep their global indices in int64_t, and a few narrow to 32 bits on
purpose inside a per-CTA or per-unit domain (os_clamp, the tiled resampler's per-thread offsets, the TMA byte counts of
the Welch kernels).  The other suites run at small sizes; this one crosses both limits.

A. Virtual global offsets.  A range call (dspb200_os_exec_range_dev, dspb200_resample_exec_range_dev,
   dspb200_welch_exec_range_dev, dspb200_welch_accumulate_dev) holds only its local window, so a global offset of 2^40
   costs no memory.  The same local data at offset O must give the result of offset 0 bit for bit, and that result is
   exact against an integer reference (overlap-save, resampling) on integer data.  The data of a window is a 64-bit
   hash of the global sample index, so any window at any offset can be regenerated on the host.  The largest offset the
   index domain of dspb200.h admits must still work; one more must be refused with DSPB200_EINVALID and no launch.
B. Real buffers over 2^31 elements and 4 GiB: one device buffer of 2^31 + 2^21 + 3 Float32 samples of integers in
   [-8, 8], filled on the device.  Results are exact against a host reference at probes around the start, the end,
   random places and both limits, and whole outputs equal (on the device) the same work issued as small calls on
   pointers into the buffer, whose indices the other suites already pin.  The buffer is refilled in place as Float64,
   ComplexF32 or ComplexF64 for the column matrices (3 FIR or resampling columns, the last past 4 GiB), and read as
   channel matrices of odd and 16-byte aligned channel lengths by the batched Welch, Welch stream, multitaper and STFT
   calls, each checked channel equal to the call on its own pointer bit for bit or within the float64 bound.  The stateful
   FIR and overlap-save forms, a resampler stream chunk over 2^31 samples after a history, and the arbitrary-rate batch
   run on it too.
C. Host pointers: the chunked host paths of fftfilt, welch_pgram and resample on a pageable array of 2^31 + 2^21 + 3
   samples.

Each test asserts that its geometry crosses the limits it is about, so that a later edit cannot shrink it below them.
The CPU tests check the hash, the sharding arithmetic at totals of 2^34 .. 2^40, the restated index domain, and that a
model of a range call whose global offsets wrap to 32 bits disagrees with the reference at every probe class: the
probes can see the defect these tests are for."""
import math

import numpy as np
import pytest

import test_os_kernel_paths as osk
import test_resample_kernel_paths as rk
import test_spectral_kernel_paths as kp
from test_os_kernel_paths import check_exact, exact_conv, int_signal, int_taps
from test_resample_kernel_paths import polyphase_ref
from test_spectral_kernel_paths import power_bound

F32, F64, C64, C128 = osk.F32, osk.F64, osk.C64, osk.C128
EINVALID = -1
INDEX_LIMIT = 1 << 61                  # DSPB200_INDEX_LIMIT, include/dspb200.h
PHASE_LIMIT = 1 << 62                  # DSPB200_PHASE_LIMIT
E31, B32 = 1 << 31, 1 << 32            # element index 2^31, byte offset 2^32
BIG_N = (1 << 31) + (1 << 21) + 3      # Float32 samples of the shared large buffer: 8 GiB + 8 MiB + 12 bytes
U64 = np.uint64


# =============================================================================== data as a function of the global index

def _mix(z):
    """splitmix64 finaliser on uint64 arrays (wrapping arithmetic)."""
    z = z ^ (z >> U64(30))
    z = z * U64(0xBF58476D1CE4E5B9)
    z = z ^ (z >> U64(27))
    z = z * U64(0x94D049BB133111EB)
    return z ^ (z >> U64(31))


def hashed(begin, n, dt, seed=0):
    """Samples [begin, begin + n) of the virtual signal: integers in [-8, 8] (both parts for complex), a hash of the
    global index, so any window at any offset (negative, or up to 2^62) can be regenerated."""
    idx = (np.arange(n, dtype=np.int64) + np.int64(begin)).astype(U64)
    base = idx * U64(2) + U64(0x9E3779B97F4A7C15) * U64(seed + 1)
    with np.errstate(over="ignore"):
        re = (_mix(base) % U64(17)).astype(np.int64) - 8
        v = re.astype(np.float64)
        if np.dtype(dt).kind == "c":
            v = v + 1j * ((_mix(base + U64(1)) % U64(17)).astype(np.int64) - 8)
    return v.astype(dt)


def probe_starts(n, width, esz, seed=0, extra=()):
    """Starts of probe windows of `width` elements over a buffer of n elements of esz bytes: the start, the end, a few
    random places, and just either side of element 2^31 and byte 2^32 (where they lie inside the buffer)."""
    rng = np.random.default_rng(seed)
    c = [0, n - width] + [int(v) for v in rng.integers(0, n - width, 4)] + list(extra)
    for limit in (E31, B32 // esz):
        if limit < n:
            c += [limit - width // 2, limit - width, limit]
    return sorted({min(max(0, v), n - width) for v in c})


# =============================================================================== the index domain, restated from dspb200.h

def _inside(v):
    return -INDEX_LIMIT <= v <= INDEX_LIMIT


def os_range_ok(u_begin, nu_local, out_begin, out_count):
    return (nu_local >= 0 and out_count >= 0 and out_begin >= 0 and _inside(u_begin) and _inside(u_begin + nu_local)
            and _inside(out_begin + out_count))


def rs_range_ok(I, D, x_begin, nx_local, n0, phi0, j_begin, nout_local):
    j_end = j_begin + nout_local
    return (nx_local >= 0 and nout_local >= 0 and j_begin >= 0 and n0 >= 0 and _inside(j_end)
            and phi0 + j_end * D <= PHASE_LIMIT and _inside(n0 + (phi0 + j_end * D) // I) and _inside(x_begin)
            and _inside(x_begin + nx_local))


def welch_range_ok(n, hop, length, sample_offset, seg_begin, seg_end):
    return (length >= 0 and 0 <= seg_begin <= seg_end and _inside(sample_offset) and _inside(sample_offset + length)
            and (seg_end == seg_begin or (seg_end - 1) * hop + n <= INDEX_LIMIT))


def _largest(ok, lo=0):
    """Largest k >= lo with ok(k), for a predicate that holds on [lo, K] and fails above."""
    assert ok(lo)
    hi = 1
    while ok(lo + hi):
        hi *= 2
    a, b = lo + hi // 2, lo + hi            # ok(a), not ok(b)
    while b - a > 1:
        m = (a + b) // 2
        a, b = (m, b) if ok(m) else (a, m)
    return a


def os_offsets(lo, hi, b, c):
    """Offsets O of one overlap-save range (stored input [lo, hi), outputs [b, b+c)): 0, either side of 2^31, past 2^32
    and 2^40, and the largest the domain admits (O + 1 is refused)."""
    top = _largest(lambda o: os_range_ok(lo + o, hi - lo, b + o, c))
    return [0, E31 - 1, E31, B32 + 1, (1 << 40) + 3, top], top + 1


def rs_shifts(I, D, lo, hi, n0, phi0, b, e):
    """Shifts k (outputs by k*I, inputs by k*D) of one resampling range: outputs across 2^31 and 2^32, inputs across
    2^31 and 2^32, and the largest the domain admits (k + 1 is refused)."""
    def ok(k):
        return rs_range_ok(I, D, lo + k * D, hi - lo, n0, phi0, b + k * I, e - b)
    ks = [0] + [max(0, (lim - (b + e) // 2) // I) for lim in (E31, B32)] + [max(0, (lim - (lo + hi) // 2) // D)
                                                                            for lim in (E31, B32)]
    top = _largest(ok)
    return ks + [top], top + 1


def welch_shifts(n, hop, b, e):
    """Shifts K (segments by K, samples by K*hop) of one Welch range [b, e): K*hop across 2^31, 2^32 and 2^40, and the
    largest the domain admits (K + 1 is refused)."""
    lo, hi = b * hop, (e - 1) * hop + n

    def ok(k):
        return welch_range_ok(n, hop, hi - lo, lo + k * hop, b + k, e + k)
    top = _largest(ok)
    return [0] + [max(0, (lim - (lo + hi) // 2) // hop) for lim in (E31, B32, 1 << 40)] + [top], top + 1


# =============================================================================== case tables

OS_FUSED = [(dt, N) for dt in (F32, C64) for N in (32, 1024, 4096, 8192, 16384)] + \
           [(dt, N) for dt in (F64, C128) for N in (32, 1024, 4096, 8192)]
OS_GENERIC = [(dt, N) for dt in (F32, F64, C64, C128) for N in (1000, 65536)]
OS_CASES = OS_FUSED + OS_GENERIC


def _rs_cases():
    """One PHASE_CASES entry per resampler family: mp2 with taps in the constant bank and in shared memory, mp, tiled
    and generic."""
    picked = {}
    for c in rk.PHASE_CASES:
        fam = rk.expected_family(*c)
        key = (fam, rk.mp2_v3(c[0], c[1], c[3], c[4])) if fam == "mp2" else (fam, None)
        picked.setdefault(key, c)
    return [picked[k] for k in sorted(picked, key=str)]


RS_CASES = _rs_cases()
# (dtype, nfft, hop): fused real and complex, 16-byte aligned hop (TMA) and not (direct loads), one cuFFT size
WELCH_CASES = [(F32, 4096, 2048), (F32, 4096, 2047), (C64, 2048, 1024), (C64, 2048, 1023), (F64, 1024, 511),
               (C128, 512, 256), (F32, 16384, 8192), (F32, 1000, 500)]


def _welch_ranges(k):
    return [(0, k), (3, 4), (5, k - 2)]


# =============================================================================== CPU

def test_hash_is_a_function_of_the_global_index():
    for dt in (F32, F64, C64, C128):
        whole = hashed(-50, 300, dt)
        for a in (-50, -1, 0, 17, 200):
            assert np.array_equal(hashed(a, 30, dt), whole[a + 50:a + 80])
        big = hashed(INDEX_LIMIT - 100, 200, dt)
        assert np.array_equal(big[100:150], hashed(INDEX_LIMIT, 50, dt))
        for v in (whole, big):
            parts = [v.real] + ([v.imag] if np.dtype(dt).kind == "c" else [])
            for p in parts:
                assert p.min() == -8 and p.max() == 8 and np.array_equal(p, np.rint(p))
    # neighbouring offsets 2^32 apart hold different data: a read that wrapped to 32 bits would see other values
    assert not np.array_equal(hashed(5, 64, F32), hashed(5 + B32, 64, F32))
    assert not np.array_equal(hashed(5, 64, F32), hashed(5 - E31 * 2, 64, F32))


def test_index_domain_restated():
    # the accepted and the refused edge of each range form sit on either side of 2^61 / 2^62
    nv, nu, ranges = osk.range_case(4096)
    for b, c in ranges:
        lo = min(nu, max(0, b - (nv - 1)))
        hi = max(lo, min(nu, b + c))
        offs, refused = os_offsets(lo, hi, b, c)
        assert offs[-1] + max(hi, b + c) == INDEX_LIMIT
        assert os_range_ok(lo + offs[-1], hi - lo, b + offs[-1], c)
        assert not os_range_ok(lo + refused, hi - lo, b + refused, c)
        assert all(o >= E31 for o in offs[2:]) and offs[1] < E31 <= offs[1] + max(hi, b + c)
    assert not os_range_ok(-INDEX_LIMIT - 1, 0, 0, 1) and os_range_ok(-INDEX_LIMIT, 5, 0, 1)
    for I, D, hlen, tx, th in RS_CASES:
        for b, e in ((1, 300), (300, 301)):
            lo, hi = 0, 400
            ks, refused = rs_shifts(I, D, lo, hi, 2, I - 1, b, e)
            top = ks[-1]
            assert rs_range_ok(I, D, lo + top * D, hi - lo, 2, I - 1, b + top * I, e - b)
            assert not rs_range_ok(I, D, lo + refused * D, hi - lo, 2, I - 1, b + refused * I, e - b)
            jD = (b + top * I) * D
            # with I > 1 the phase reaches 2^62 (j*D close to the phase limit), with I == 1 the input index 2^61 binds
            assert jD > (PHASE_LIMIT if I > 1 else INDEX_LIMIT) // (2 * max(I, D)), (I, D, jD)
            # the middle of the outputs, then of the inputs, lies at 2^31 and at 2^32
            for k, lim in zip(ks[1:3], (E31, B32)):
                assert abs((b + e) // 2 + k * I - lim) <= I
            for k, lim in zip(ks[3:5], (E31, B32)):
                assert abs((lo + hi) // 2 + k * D - lim) <= D
    for dt, N, hop in WELCH_CASES:
        k = 20
        for b, e in _welch_ranges(k):
            Ks, refused = welch_shifts(N, hop, b, e)
            lo, hi = b * hop, (e - 1) * hop + N
            assert welch_range_ok(N, hop, hi - lo, lo + Ks[-1] * hop, b + Ks[-1], e + Ks[-1])
            assert not welch_range_ok(N, hop, hi - lo, lo + refused * hop, b + refused, e + refused)
            for K, lim in zip(Ks[1:4], (E31, B32, 1 << 40)):
                assert lo + K * hop < lim < hi + K * hop + hop, (dt, N, hop, b, e, K)


def _brute_conv_shard(nu, nv, nout, world, rank, align):
    # every output belongs to exactly one rank, contiguous in rank order; outputs m read inputs [m - nv + 1, m]
    nblk = -(-nout // align)
    per = [nblk // world + (1 if r < nblk % world else 0) for r in range(world)]
    b = min(nout, sum(per[:rank]) * align)
    e = min(nout, sum(per[:rank + 1]) * align)
    return b, e, (max(0, b - (nv - 1)), max(0, min(nu, e)))


@pytest.mark.parametrize("total_log2", [34, 36, 38, 40])
def test_sharding_at_large_totals(total_log2):
    from dspb200 import sharding as sh
    total, world = (1 << total_log2) + 12345, 16
    rng = np.random.default_rng(total_log2)
    ranks = sorted({0, world - 1} | {int(r) for r in rng.integers(0, world, 4)})
    for nv, align in ((4097, 1), (4097, 12288), (257, 16384 - 256)):
        nout = total + nv - 1
        ends = []
        for r in range(world):
            s = sh.conv_shard(total, nv, nout, world, r, align)
            ends.append((s.out_begin, s.out_begin + s.out_count))
            if r in ranks:
                b, e, (ib, ie) = _brute_conv_shard(total, nv, nout, world, r, align)
                assert (s.out_begin, s.out_begin + s.out_count, s.in_begin, s.in_end) == (b, e, ib, ie)
                assert b % align == 0
        assert ends[0][0] == 0 and ends[-1][1] == nout and all(a[1] == c[0] for a, c in zip(ends, ends[1:]))
    for n, hop in ((4096, 2048), (4096, 2047), (1000, 1000)):
        k = (total - n) // hop + 1
        segs = []
        for r in range(world):
            s = sh.welch_stream_shard(total, n, n - hop, world, r)
            assert s.k_total == k
            segs.append((s.seg_begin, s.seg_end))
            if r in ranks and s.seg_end > s.seg_begin:
                lo, hi = sh.split_range(total, world, r)
                # brute force around the edges: the first segment starts in [lo, hi), its predecessor before lo; the
                # last one starts in range, its successor at or past hi (or past the last segment)
                assert lo <= s.seg_begin * hop < hi and (s.seg_begin == 0 or (s.seg_begin - 1) * hop < lo)
                assert lo <= (s.seg_end - 1) * hop < hi and (s.seg_end == k or s.seg_end * hop >= hi)
                assert (s.sample_begin, s.sample_end) == (s.seg_begin * hop, (s.seg_end - 1) * hop + n)
        assert segs[0][0] == 0 and segs[-1][1] == k and all(a[1] == c[0] for a, c in zip(segs, segs[1:]))
    for I, D, tpp in ((3, 2, 13), (1, 4, 40), (160, 147, 8)):
        nx = total
        nout = nx * I // D
        n0, phi0 = 7, I - 1
        for r in ranks:
            s = sh.resample_shard(nx, nout, I, D, n0, phi0, tpp, world, r)
            b, e = sh.split_range(nout, world, r)
            assert (s.j_begin, s.j_begin + s.out_count) == (b, e)
            # the windows of the first and the last output, from the definition p = phi0 + j*D, n = n0 + p // I
            first = n0 + (phi0 + b * D) // I - (tpp - 1)
            last = n0 + (phi0 + (e - 1) * D) // I
            assert s.in_begin == max(0, first) and s.in_end == max(0, min(nx, last + 1))
            assert last > E31 or r == 0


# ---- the checks can fail: ranges whose global offsets wrap to 32 bits

def _wrap_i32(v):
    return ((int(v) + E31) % B32) - E31


def _os_model(u_window, lo, v, b, c, wrap):
    """out[m], m in [b, b+c), of the virtual signal holding u_window at [lo, ...): the slot's global input index
    computed in 64 bits, or narrowed to int32 (wrap) before the local index is formed."""
    nv = v.size
    out = np.zeros(c, dtype=np.complex128)
    for i, m in enumerate(range(b, b + c)):
        for t in range(nv):
            g = m - t
            g = _wrap_i32(g) if wrap else g
            li = g - lo
            if 0 <= li < u_window.size:
                out[i] += u_window[li] * v[t]
    return out


def _rs_model(x_window, x_begin, h, I, D, n0, phi0, j_begin, nout, wrap):
    tpp = -(-h.size // I)
    hp = np.zeros(tpp * I)
    hp[:h.size] = h
    out = np.zeros(nout, dtype=np.complex128)
    for i in range(nout):
        j = j_begin + i
        p = phi0 + j * D
        p = _wrap_i32(p) if wrap else p
        n, phi = n0 + p // I, p % I
        for t in range(tpp):
            li = n - t - x_begin
            if 0 <= li < x_window.size:
                out[i] += hp[phi + t * I] * x_window[li]
    return out


def _welch_model(buf, sample_offset, seg, hop, n, wrap):
    """The samples a Welch unit loads for segment `seg`: byte offset of the segment from the buffer start, in 64 bits
    or narrowed to uint32 (wrap).  buf is a function of the local index."""
    byte = (seg * hop - sample_offset) * 4
    if wrap:
        byte %= B32
    return buf(byte // 4, n)


def test_probes_detect_offsets_wrapped_to_32_bits():
    rng = np.random.default_rng(3)
    # overlap-save: a range at offset O against the reference (the O = 0 twin of the same local data)
    v = int_taps(rng, 33, F64)
    lo, b, c = 100, 140, 50
    win = hashed(lo, 200, F64)
    want = exact_conv(win, v)[b - lo:b - lo + c]
    for O in (E31, B32 + 1, (1 << 40) + 3, INDEX_LIMIT - 400):
        assert np.array_equal(_os_model(win, lo + O, v, b + O, c, False), want)
        assert not np.array_equal(_os_model(win, lo + O, v, b + O, c, True), want), O
    # a range across 2^31 - 1: only its outputs past the limit go wrong, and they do
    O = E31 - 1 - (b + c // 2)
    bad = _os_model(win, lo + O, v, b + O, c, True) != want
    assert bad[c // 2 + 1:].all() and not bad[:c // 2 + 1].any()
    # resampling: shifted by k (outputs by k*I, inputs by k*D)
    I, D, hlen = 3, 2, 38
    h = rk.int_taps(rng, hlen, F64)
    xw = hashed(0, 400, F64)
    n0, phi0, j_b, cnt = 2, 2, 40, 30
    want = polyphase_ref(xw, h, I, D, n0, phi0, j_b + cnt)[j_b:]
    for k in ((E31 - 100) // I, B32 // I + 1, (1 << 40) // I, (PHASE_LIMIT // D - 500) // I):
        assert np.array_equal(_rs_model(xw, k * D, h, I, D, n0, phi0, j_b + k * I, cnt, False), want)
        assert not np.array_equal(_rs_model(xw, k * D, h, I, D, n0, phi0, j_b + k * I, cnt, True), want), k
    # Welch: the samples a segment loads, with its byte offset in 64 bits or in a uint32
    n, hop = 64, 32
    for K in (E31 // hop, B32 // hop + 1, (1 << 40) // hop + 3, (INDEX_LIMIT - 4096) // hop):
        def local(i, m):
            return hashed(K * hop + i, m, F32)
        for seg_rel in (0, 5, (B32 // 4) // hop + 1):            # the last one lies 4 GiB into the local buffer
            right = _welch_model(local, K * hop, K + seg_rel, hop, n, False)
            assert np.array_equal(right, hashed((K + seg_rel) * hop, n, F32))
        wrong = _welch_model(local, K * hop, K + (B32 // 4) // hop + 1, hop, n, True)
        assert not np.array_equal(wrong, right), K
    # the element and byte probes of the large buffer: a 32-bit element index or byte offset reads another sample
    for esz in (4, 8, 16):
        n_el = BIG_N * 4 // esz
        starts = probe_starts(n_el, 64, esz)
        past = [s for s in starts if s * esz >= B32]
        assert past, esz
        for s in past:
            idx = np.arange(s, s + 64)
            wrapped = idx * esz % B32 // esz
            assert not np.array_equal(hashed(wrapped[0], 64, F32), hashed(s, 64, F32)), (esz, s)
        if esz == 4:
            for s in (s for s in starts if s + 64 > E31):
                idx = [_wrap_i32(i) for i in range(s, s + 64)]
                assert not np.array_equal(hashed(0, 64, F32) * 0 + [hashed(i, 1, F32)[0] for i in idx],
                                          hashed(s, 64, F32)), s


def test_large_buffer_geometry():
    # the shared buffer crosses element 2^31 as Float32 and byte 2^32 as every eltype, with room to spare
    assert BIG_N > E31 and BIG_N * 4 > B32
    for esz in (8, 16):
        assert BIG_N * 4 // esz * esz > B32
    for esz in (4, 8, 16):
        starts = probe_starts(BIG_N * 4 // esz, 64, esz)
        assert any(s * esz < B32 <= (s + 64) * esz for s in starts)
        if esz == 4:
            assert any(s < E31 <= s + 64 for s in starts)
    # the overlap-save twins are cut at multiples of a block pair; the Welch shards at segment boundaries
    for nfft, nv in LARGE_OS:
        L = nfft - nv + 1
        cuts = _os_twin_cuts(BIG_N, L)
        assert cuts[0] == 0 and cuts[-1] == BIG_N and all(c % (2 * L) == 0 for c in cuts[1:-1])
        assert any(a < E31 <= b for a, b in zip(cuts, cuts[1:]))


# =============================================================================== GPU helpers

@pytest.fixture(scope="module")
def dsp():
    return pytest.importorskip("dspb200")


def _refused(dsp, call):
    """call() raises DSPB200Error(EINVALID) and launches nothing."""
    n0 = dsp.launch_count()
    with pytest.raises(dsp._lib.DSPB200Error) as e:
        call()
    assert e.value.code == EINVALID and dsp.launch_count() == n0


def _bits(a):
    return kp._bits(a)


# =============================================================================== GPU, A: virtual global offsets

@pytest.mark.gpu
@pytest.mark.parametrize("dt,N", OS_CASES, ids=[f"{dt.name}-{N}" for dt, N in OS_CASES])
def test_os_range_at_global_offsets(dsp, dt, N):
    from dspb200 import device
    rng = np.random.default_rng([N, dt.num, 40])
    nv, nu, ranges = osk.range_case(N)
    taps = int_taps(rng, nv, dt)
    plan = osk._plan(dsp, taps, N)
    try:
        assert plan.fused == (N in (32, 1024, 4096, 8192, 16384))
        f64 = osk._f64(dt)
        u = hashed(0, nu, dt)
        full = exact_conv(u, taps, nu + nv - 1 + 4 * N)
        for b, c in ranges:
            lo = min(nu, max(0, b - (nv - 1)))
            hi = max(lo, min(nu, b + c))
            gu = osk.Guarded(dt, hi - lo, rng=rng, data=u[lo:hi])
            offs, refused = os_offsets(lo, hi, b, c)
            first = None
            for O in offs:
                go = osk.Guarded(dt, c)
                plan.exec_range_dev(gu.ptr, lo + O, hi - lo, go.ptr, b + O, c, 0)
                device.sync()
                gu.data()
                y = go.data()
                if first is None:
                    first = y
                    check_exact(y, full[b:b + c], f64, what=(b, c))
                assert np.array_equal(_bits(y), _bits(first)), (b, c, O)
                # hashed data at the offset itself: exact against the integer convolution of that window
                if O:
                    w = hashed(lo + O, hi - lo, dt)
                    gw = osk.Guarded(dt, hi - lo, rng=rng, data=w)
                    go2 = osk.Guarded(dt, c)
                    plan.exec_range_dev(gw.ptr, lo + O, hi - lo, go2.ptr, b + O, c, 0)
                    device.sync()
                    want = np.zeros(c, dtype=np.complex128 if osk._cplx(dt) else np.float64)
                    if hi > lo:
                        cw = exact_conv(w, taps)
                        s = b - lo
                        take = cw[max(0, s):s + c]
                        want[max(0, -s):max(0, -s) + take.size] = take
                    check_exact(go2.data(), want, f64, what=("hashed", b, c, O))
            go = osk.Guarded(dt, c)
            _refused(dsp, lambda: plan.exec_range_dev(gu.ptr, lo + refused, hi - lo, go.ptr, b + refused, c, 0))
            go.data()
        # stored input more than 2^31 samples before or after the outputs: every output is zero (a block without stored
        # samples is transformed like any other, so its zeros may carry either sign, as dspb200.h states)
        b, c = osk.range_case(N)[2][3]
        w = hashed(0, 3 * N, dt)
        gw = osk.Guarded(dt, w.size, rng=rng, data=w)
        for O in (0, B32 + 1, (1 << 40) + 3):
            for u_begin in (b + O - E31 - 1 - w.size, b + O + c + E31 + 1):
                go = osk.Guarded(dt, c)
                plan.exec_range_dev(gw.ptr, u_begin, w.size, go.ptr, b + O, c, 0)
                device.sync()
                y = go.data()
                assert np.all(y == 0), (O, u_begin)
        go = osk.Guarded(dt, 1)
        _refused(dsp, lambda: plan.exec_range_dev(gw.ptr, -INDEX_LIMIT - 1, w.size, go.ptr, 0, 1, 0))
        _refused(dsp, lambda: plan.exec_range_dev(gw.ptr, 0, INDEX_LIMIT + 1, go.ptr, 0, 1, 0))
        _refused(dsp, lambda: plan.exec_range_dev(gw.ptr, 0, w.size, go.ptr, INDEX_LIMIT, 1, 0))
        go.data()
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("I,D,hlen,tx,th", RS_CASES, ids=[rk._case_id(c) for c in RS_CASES])
def test_resample_range_at_global_offsets(dsp, I, D, hlen, tx, th):
    from dspb200 import device
    fam = rk.expected_family(I, D, hlen, tx, th)
    tpp = -(-hlen // I)
    T = rk.tile_outputs(fam, I, D, tx, th)
    nout = 3 * T + 11
    nx = math.ceil(nout * D / I)
    n0, phi0 = 2, I - 1
    rng = np.random.default_rng([I, D, hlen, 40])
    h = rk.int_taps(rng, hlen, th)
    x = hashed(0, nx, tx)
    want = polyphase_ref(x, h, I, D, n0, phi0, nout)
    plan = dsp._lib.ResamplePlan(tx, h, I, D)
    try:
        for b, e in ((1, T + 2), (T + 2, T + 3 + T // 2), (2 * T + 1, nout)):
            lo = max(0, n0 + (phi0 + b * D) // I - (tpp - 1))
            hi = max(lo, min(nx, n0 + (phi0 + (e - 1) * D) // I + 1))
            local = device.to_device(x[lo:hi])
            ks, refused = rs_shifts(I, D, lo, hi, n0, phi0, b, e)
            first = None
            for k in ks:
                part = device.DeviceArray((e - b,), plan.out_dtype)
                plan.exec_range_dev(local.ptr, lo + k * D, hi - lo, n0, phi0, part.ptr, b + k * I, e - b, 0)
                device.sync()
                y = part.to_host()
                if first is None:
                    first = y
                    assert np.array_equal(y, want[b:e]), (fam, b, e)
                assert np.array_equal(_bits(y), _bits(first)), (fam, b, e, k)
            part = device.DeviceArray((e - b,), plan.out_dtype)
            _refused(dsp, lambda: plan.exec_range_dev(local.ptr, lo + refused * D, hi - lo, n0, phi0, part.ptr,
                                                      b + refused * I, e - b, 0))
        _refused(dsp, lambda: plan.exec_range_dev(local.ptr, 0, hi - lo, INDEX_LIMIT + 1, phi0, part.ptr, 0, 1, 0))
        _refused(dsp, lambda: plan.exec_range_dev(local.ptr, -INDEX_LIMIT - 1, hi - lo, n0, phi0, part.ptr, 0, 1, 0))
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,N,hop", WELCH_CASES, ids=[f"{dt.name}-{N}-hop{hop}" for dt, N, hop in WELCH_CASES])
def test_welch_range_at_global_offsets(dsp, dt, N, hop):
    from dspb200 import device
    rng = np.random.default_rng([N, hop, dt.num, 40])
    n = N
    k = 20
    length = (k - 1) * hop + n
    x = hashed(0, length, dt)
    onesided = not kp._cplx(dt)
    w = kp.window_of("hann", n, rng)
    r = k * kp.norm2_of(w, n)
    plan = kp._plan(dsp, dt, n, hop, N, onesided, w)
    nout = plan.nout
    try:
        X, en = kp.ref_segments(x, n, hop, N, w)
        for b, e in _welch_ranges(k):
            lo, hi = b * hop, (e - 1) * hop + n
            g = kp.Guarded(dt, hi - lo, rng, x[lo:hi])
            Ks, refused = welch_shifts(n, hop, b, e)
            first = None
            for K in Ks:
                go = kp.Guarded(kp._real(dt), nout)
                plan.welch_range_dev(g.ptr, hi - lo, lo + K * hop, b + K, e + K, r, go.ptr, 0)
                # begin / accumulate in two pieces / finalize on the same buffer
                gs = kp.Guarded(kp._real(dt), nout)
                m = (b + e) // 2
                plan.welch_begin_dev(0)
                plan.welch_accumulate_dev(g.ptr, hi - lo, lo + K * hop, b + K, m + K, 0)
                plan.welch_accumulate_dev(g.ptr, hi - lo, lo + K * hop, m + K, e + K, 0)
                plan.welch_finalize_dev(r, gs.ptr, 0)
                device.sync()
                g.data()
                P, Ps = go.data(), gs.data()
                if first is None:
                    first = (P, Ps)
                    Xs = X[b:e]
                    kp.check_welch(P, Xs, en[b:e], N, onesided, r, kp.eps(dt), e - b, (b, e))
                assert kp.same_bits(P, first[0]) and kp.same_bits(Ps, first[1]), (b, e, K)
            go = kp.Guarded(kp._real(dt), nout)
            _refused(dsp, lambda: plan.welch_range_dev(g.ptr, hi - lo, lo + refused * hop, b + refused, e + refused, r,
                                                       go.ptr, 0))
            _refused(dsp, lambda: plan.welch_accumulate_dev(g.ptr, hi - lo, lo + refused * hop, b + refused,
                                                            e + refused, 0))
        _refused(dsp, lambda: plan.welch_accumulate_dev(g.ptr, -1, 0, 0, 0, 0))
        _refused(dsp, lambda: plan.welch_accumulate_dev(g.ptr, 10, -INDEX_LIMIT - 1, 0, 0, 0))
    finally:
        plan.close()
        device.empty_cache()


# =============================================================================== GPU, B: buffers over 2^31 elements and 4 GiB

LARGE_OS = [(16384, 4097), (16384, 257), (4096, 257), (65536, 4097)]
TWIN_CHUNK = 1 << 28


def _os_twin_cuts(n, L):
    step = TWIN_CHUNK // (2 * L) * (2 * L)
    return list(range(0, n, step)) + [n]


TORCH_DT = {F32: "float32", F64: "float64", C64: "complex64", C128: "complex128"}
REAL_OF = {F32: F32, F64: F64, C64: F32, C128: F64}


class Big:
    """The shared buffer: BIG_N Float32 cells, refilled in place on the device with seeded integers in [-8, 8] for the
    eltype a test asks for (both parts for complex), so that no 8 GiB host array is needed."""

    def __init__(self, torch, buf):
        self.torch, self.buf, self.dt = torch, buf, None
        self.base_reserved = torch.cuda.memory_reserved()

    def typed(self, dt):
        """(tensor of eltype dt over the buffer, its element count)."""
        torch = self.torch
        dt = np.dtype(dt)
        n = BIG_N * 4 // dt.itemsize
        raw = self.buf[:n * dt.itemsize // 4]
        if self.dt != dt:
            gen = torch.Generator(device="cuda")
            gen.manual_seed(2024 + dt.num)
            (raw if REAL_OF[dt] == F32 else raw.view(torch.float64)).random_(-8, 9, generator=gen)
            torch.cuda.synchronize()
            self.dt = dt
        return raw.view(getattr(torch, TORCH_DT[dt])), n


@pytest.fixture(scope="module")
def big(dsp):
    """One device buffer of BIG_N Float32 samples, reused by every test of part B; freed with the library's and torch's
    pooled blocks at the end, where the peak device memory the module reserved is printed."""
    torch = pytest.importorskip("torch")
    from dspb200 import device
    nbytes = BIG_N * 4
    torch.cuda.reset_peak_memory_stats()
    try:
        buf = torch.empty(BIG_N, dtype=torch.float32, device="cuda")
    except torch.OutOfMemoryError:
        pytest.skip(f"the shared GPU has no room for {nbytes} bytes")
    big = Big(torch, buf)
    big.typed(F32)
    yield big
    print(f"\npeak device memory reserved by the large-buffer tests (torch allocations; plan scratch not included): "
          f"{torch.cuda.max_memory_reserved() / 2**30:.2f} GiB on {torch.cuda.get_device_name()}")
    del buf, big
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    device.empty_cache()


def _alloc(torch, n, dtype):
    if isinstance(dtype, np.dtype):
        dtype = getattr(torch, TORCH_DT[dtype])
    try:
        return torch.empty(n, dtype=dtype, device="cuda")
    except torch.OutOfMemoryError:
        pytest.skip(f"the shared GPU has no room for {n * torch.empty(0, dtype=dtype).element_size()} bytes")


def _host(t, a, b):
    return t[a:b].cpu().numpy()


def _free(torch, *plans):
    from dspb200 import device
    for p in plans:
        p.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("nb", [9, 257])
def test_fir_over_2e31_samples(dsp, big, nb):
    torch = big.torch
    buf, _ = big.typed(F32)
    from dspb200 import device
    rng = np.random.default_rng(nb)
    b = int_taps(rng, nb, F32)
    plan = dsp._lib.FirPlan(b)
    out = _alloc(torch, BIG_N, torch.float32)
    try:
        assert BIG_N > E31 and BIG_N * 4 > B32
        plan.exec_dev(buf.data_ptr(), BIG_N, 1, out.data_ptr(), 0)
        device.sync()
        W = 64
        for s in probe_starts(BIG_N, W, 4, seed=nb):
            a = max(0, s - (nb - 1))
            xw = _host(buf, a, s + W).astype(np.float64)
            want = np.convolve(xw, b.astype(np.float64))[s - a:s - a + W]
            got = _host(out, s, s + W)
            assert np.array_equal(got.astype(np.float64), want), s
    finally:
        plan.close()
        del out
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("nfft,nv", LARGE_OS, ids=[f"nfft{a}-nv{b}" for a, b in LARGE_OS])
def test_os_over_2e31_samples(dsp, big, nfft, nv):
    torch = big.torch
    buf, _ = big.typed(F32)
    from dspb200 import device
    rng = np.random.default_rng([nfft, nv])
    v = int_taps(rng, nv, F32)
    plan = osk._plan(dsp, v, nfft)
    assert plan.fused == (nfft <= 16384)
    L = nfft - nv + 1
    out = _alloc(torch, BIG_N, torch.float32)
    twin = _alloc(torch, TWIN_CHUNK + 2 * L, torch.float32)
    try:
        plan.exec_dev(buf.data_ptr(), BIG_N, 1, out.data_ptr(), BIG_N, 0)
        device.sync()
        W = 64
        for s in probe_starts(BIG_N, W, 4, seed=nfft + nv):
            a = max(0, s - (nv - 1))
            xw = _host(buf, a, s + W)
            want = exact_conv(xw, v)[s - a:s - a + W]
            check_exact(_host(out, s, s + W), want, False, what=("probe", s))
        # the whole output against range twins on pointers into the buffer: local indices only, the same blocks
        cuts = _os_twin_cuts(BIG_N, L)
        for m0, m1 in zip(cuts, cuts[1:]):
            i0 = max(0, m0 - (nv - 1))
            i1 = min(BIG_N, m1 + 2 * nfft)            # every sample the big call's blocks of these outputs hold
            plan.exec_range_dev(buf.data_ptr() + 4 * i0, i0 - m0, i1 - i0, twin.data_ptr(), 0, m1 - m0, 0)
            device.sync()
            assert torch.equal(out[m0:m1], twin[:m1 - m0]), (m0, m1)
    finally:
        plan.close()
        del out, twin
        torch.cuda.empty_cache()
        device.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt,hop", [(F32, 2048), (F32, 2047), (C64, 2048), (C64, 2047)],
                         ids=["f32-aligned", "f32-unaligned", "c64-aligned", "c64-unaligned"])
def test_welch_over_4gib(dsp, big, dt, hop):
    # one signal over the whole buffer (ComplexF32: 2^30 samples, 8 GiB) against the sum of shard calls on
    # pointer-offset local buffers; the partition into virtual CTAs differs, so within the bound at m = all segments
    torch = big.torch
    buf, _ = big.typed(F32)
    from dspb200 import device, sharding
    n = N = 4096
    esz = dt.itemsize
    length = BIG_N * 4 // esz
    assert length * esz > B32 and (dt != F32 or length > E31)
    plan = kp._plan(dsp, dt, n, hop, N, dt == F32, None)
    k = plan.nsegments(length)
    r = float(k * n)
    nout = plan.nout
    try:
        one = device.DeviceArray((nout,), F32)
        plan.welch_dev(buf.data_ptr(), length, r, one.ptr, 0)
        piece = device.DeviceArray((nout,), F32)
        plan.welch_begin_dev(0)
        plan.welch_accumulate_dev(buf.data_ptr(), length, 0, 0, k // 2, 0)
        plan.welch_accumulate_dev(buf.data_ptr(), length, 0, k // 2, k, 0)
        plan.welch_finalize_dev(r, piece.ptr, 0)
        device.sync()
        one, piece = one.to_host().astype(np.float64), piece.to_host().astype(np.float64)
        total = np.zeros(nout)
        part = device.DeviceArray((nout,), F32)
        world = 8
        for rank in range(world):
            s = sharding.welch_stream_shard(length, n, n - hop, world, rank)
            if s.seg_end == s.seg_begin:
                continue
            plan.welch_range_dev(buf.data_ptr() + esz * s.sample_begin, s.sample_end - s.sample_begin, 0, 0,
                                 s.seg_end - s.seg_begin, r, part.ptr, 0)
            device.sync()
            total += part.to_host()
        mult = np.ones(nout) if dt == C64 else kp.bins_and_mult(N, True)[1]
        S = total * r / k / mult                   # the mean segment power of the shards, as the reference spectrum
        E = n * (128.0 if dt == C64 else 64.0)     # a segment's energy is at most n |x|max^2
        for P in (one, piece):
            err = np.abs(P * r / k / mult - S)
            assert np.all(err <= power_bound(S, E, kp.eps(dt), N, k)), (dt, hop)
        assert np.all(np.isfinite(one)) and one.min() > 0
    finally:
        plan.close()
        device.empty_cache()


@pytest.mark.gpu
def test_resample_decimating_over_2e31_samples(dsp, big):
    torch = big.torch
    buf, _ = big.typed(F32)
    from dspb200 import device
    I, D, hlen = 1, 4, 40
    rng = np.random.default_rng(7)
    h = rk.int_taps(rng, hlen, F32)
    plan = dsp._lib.ResamplePlan(F32, h, I, D)
    nout = -(-BIG_N * I // D)
    n0, phi0 = 5, 0
    assert (nout - 1) * D + n0 > E31 and BIG_N * 4 > B32
    out = _alloc(torch, nout, torch.float32)
    try:
        plan.exec_dev(buf.data_ptr(), BIG_N, 1, n0, phi0, out.data_ptr(), nout, 0)
        device.sync()
        W = 64
        for s in probe_starts(nout, W, 4, seed=11, extra=[(E31 - n0) // D - W // 2, (B32 // 4 - n0) // D - W // 2]):
            a = max(0, n0 + s * D - (hlen - 1))
            bnd = min(BIG_N, n0 + (s + W) * D + 1)
            xw = _host(buf, a, bnd)
            # outputs s .. s+W-1 of the whole call are outputs (s - j_a) of a call on the window with n0 shifted by a
            want = polyphase_ref(xw, h, I, D, n0 + s * D - a, phi0, W)
            assert np.array_equal(_host(out, s, s + W).astype(np.float64), want), s
    finally:
        plan.close()
        del out
        torch.cuda.empty_cache()



# ---- column matrices, stateful and streaming forms: per-column strides and byte offsets past 4 GiB

def col_probes(nx, ncols, esz, W):
    """(column, start) of probe windows of W samples in an nx x ncols column-major matrix of esz-byte elements: both ends
    of the first and the last column, and the windows around element 2^31 and byte 2^32 with the ends of the columns they
    fall in and of the column before."""
    p = {(0, 0), (0, nx - W), (ncols - 1, 0), (ncols - 1, nx - W)}
    for e in (E31, B32 // esz):
        if e < nx * ncols:
            c, i = divmod(e, nx)
            p |= {(c, min(max(0, i - W // 2), nx - W)), (c, 0), (c, nx - W)}
            if c > 0:
                p.add((c - 1, nx - W))
    return sorted(p)


def limit_cols(length, nchan, esz):
    """Channels of a length x nchan matrix to check whole: the first, the last, and those on both sides of element 2^31
    and byte 2^32."""
    c = {0, nchan - 1}
    for e in (E31, B32 // esz):
        if e < length * nchan:
            c |= {e // length - 1, e // length, e // length + 1}
    return sorted(v for v in c if 0 <= v < nchan)


def _wide(dt):
    return np.complex128 if np.dtype(dt).kind == "c" else np.float64


def rs_probe_want(read, nxc, h, I, D, n0, phi0, j_s, W):
    """Outputs j_s .. j_s+W-1 of the polyphase sum over a column of nxc samples of which read(a, b) returns [a, b)."""
    tpp = -(-h.size // I)
    p_s = phi0 + j_s * D
    a = max(0, n0 + p_s // I - (tpp - 1))
    b = max(a, min(nxc, n0 + (phi0 + (j_s + W - 1) * D) // I + 1))
    return polyphase_ref(read(a, b), h, I, D, n0 + p_s // I - a, p_s % I, W)


def test_column_probes_cross_the_limits():
    for dt, ncols in ((F64, 3), (C64, 3), (C128, 3), (F32, 1)):
        n = BIG_N * 4 // dt.itemsize
        nx = n // ncols
        pr = col_probes(nx, ncols, dt.itemsize, 64)
        assert any((c * nx + i) * dt.itemsize < B32 <= (c * nx + i + 64) * dt.itemsize for c, i in pr)
        if ncols == 3:
            assert 2 * nx * dt.itemsize > B32                          # the last column starts past 4 GiB
    for length in (MATRIX_LENS[0], MATRIX_LENS[1]):
        nchan = BIG_N // length
        cols = limit_cols(length, nchan, 4)
        assert any(c * length < E31 <= (c + 1) * length for c in cols)
        assert any(c * length * 4 < B32 <= (c + 1) * length * 4 for c in cols)
        assert any(c * length >= E31 for c in cols)


MATRIX_LENS = ((1 << 20) + 1, (1 << 20) + 4)          # an odd channel length (direct loads), a 16-byte aligned one (TMA)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, C64, C128], ids=lambda d: d.name)
def test_fir_matrix_and_state_over_4gib(dsp, big, dt):
    from dspb200 import device
    torch = big.torch
    x, n_el = big.typed(dt)
    ncols, nb, W, esz = 3, 33, 64, dt.itemsize
    nx = n_el // ncols
    assert 2 * nx * esz > B32
    rng = np.random.default_rng([dt.num, 50])
    b = int_taps(rng, nb, dt)
    w = _wide(dt)
    plan = dsp._lib.FirPlan(b)
    out = _alloc(torch, nx * ncols, dt)
    try:
        def check(si):
            for c, i in col_probes(nx, ncols, esz, W):
                a = max(0, i - (nb - 1))
                want = np.convolve(_host(x, c * nx + a, c * nx + i + W).astype(w), b.astype(w))[i - a:i - a + W]
                if si is not None and i < nb - 1:
                    m = min(W, nb - 1 - i)
                    want[:m] += si[i:i + m, c]
                assert np.array_equal(_host(out, c * nx + i, c * nx + i + W), want), (c, i)
        plan.exec_dev(x.data_ptr(), nx, ncols, out.data_ptr(), 0)
        device.sync()
        check(None)
        si = np.asfortranarray(int_signal(rng, (nb - 1, ncols), dt))
        d_si = device.to_device(si)
        d_so = device.DeviceArray((nb - 1, ncols), dt)
        plan.exec_state_dev(x.data_ptr(), nx, ncols, d_si.ptr, d_so.ptr, out.data_ptr(), 0)
        device.sync()
        check(si)
        so = d_so.to_host()
        for c in range(ncols):
            tail = _host(x, c * nx + nx - (nb - 1), c * nx + nx).astype(w)
            assert np.array_equal(so[:, c], np.convolve(tail, b.astype(w))[nb - 1:2 * (nb - 1)]), c
    finally:
        del out
        _free(torch, plan)


@pytest.mark.gpu
def test_os_state_over_2e31_samples(dsp, big):
    from dspb200 import device
    torch = big.torch
    x, nx = big.typed(F32)
    rng = np.random.default_rng(51)
    nv, W = 257, 64
    v = int_taps(rng, nv, F32)
    plan = dsp._lib.OsPlan(v, 0)
    assert plan.fused
    out = _alloc(torch, nx, F32)
    try:
        si = int_signal(rng, nv - 1, F32)
        d_si = device.to_device(si)
        d_so = device.DeviceArray((nv - 1,), F32)
        plan.exec_state_dev(x.data_ptr(), nx, 1, d_si.ptr, d_so.ptr, out.data_ptr(), 0)
        device.sync()
        for i in probe_starts(nx, W, 4, seed=51):
            a = max(0, i - (nv - 1))
            want = exact_conv(_host(x, a, i + W), v)[i - a:i - a + W]
            if i < nv - 1:
                m = min(W, nv - 1 - i)
                want[:m] += si[i:i + m]
            check_exact(_host(out, i, i + W), want, False, what=("probe", i))
        tail = _host(x, nx - (nv - 1), nx)
        check_exact(d_so.to_host(), exact_conv(tail, v)[nv - 1:2 * (nv - 1)], False, what="final state")
    finally:
        del out
        _free(torch, plan)


@pytest.mark.gpu
def test_resample_matrix_over_4gib(dsp, big):
    # a rational plan on three Float64 columns, the last starting past 4 GiB, exact at probes of every column
    from dspb200 import device
    torch = big.torch
    x, n_el = big.typed(F64)
    I, D, hlen, ncols, W = 2, 3, 25, 3, 64
    nx = n_el // ncols
    n0, phi0 = rk._resample_phase(hlen, I)
    h = rk.int_taps(np.random.default_rng(52), hlen, F64)
    plan = dsp._lib.ResamplePlan(F64, h, I, D)
    nout = nx * I // D
    out = _alloc(torch, nout * ncols, F64)
    try:
        plan.exec_dev(x.data_ptr(), nx, ncols, n0, phi0, out.data_ptr(), nout, 0)
        device.sync()
        for c, i in col_probes(nx, ncols, 8, W):
            j = min(max(0, (i - n0) * I // D), nout - W)
            want = rs_probe_want(lambda a, b: _host(x, c * nx + a, c * nx + b), nx, h, I, D, n0, phi0, j, W)
            assert np.array_equal(_host(out, c * nout + j, c * nout + j + W), want), (c, j)
    finally:
        del out
        _free(torch, plan)


@pytest.mark.gpu
def test_resample_stream_chunk_over_2e31_samples(dsp, big):
    # one chunk of 2^31 + 2^21 + 3 samples after a non-empty history: the virtual column [history; x]
    from dspb200 import device
    torch = big.torch
    x, nx = big.typed(F32)
    I, D, hlen, W = 2, 3, 25, 64
    tpp = -(-hlen // I)
    H = tpp - 1
    rng = np.random.default_rng(53)
    h = rk.int_taps(rng, hlen, F32)
    hist = int_signal(rng, H, F32)
    plan = dsp._lib.ResamplePlan(F32, h, I, D)
    deficit, phi0 = 1, 0
    nout = ((nx - deficit) * I - phi0) // D + 1
    n0v = H + deficit - 1                               # newest sample of output 0, in the virtual column
    out = _alloc(torch, nout, F32)
    try:
        d_hi = device.to_device(hist)
        d_ho = device.DeviceArray((H,), F32)
        plan.stream_exec_dev(d_hi.ptr, d_ho.ptr, x.data_ptr(), nx, 1, deficit, phi0, out.data_ptr(), nout, nout, 0)
        device.sync()
        assert np.array_equal(d_ho.to_host(), _host(x, nx - H, nx))

        def read(a, b):
            return np.concatenate([hist[a:min(b, H)], _host(x, max(a, H) - H, max(b, H) - H)])
        starts = [0, nout - W] + [min(nout - W, max(0, (e + H - n0v) * I // D - W // 2)) for e in (E31, B32 // 4)]
        for j in starts:
            want = rs_probe_want(read, H + nx, h, I, D, n0v, phi0, j, W)
            assert np.array_equal(_host(out, j, j + W), want), j
    finally:
        del out
        _free(torch, plan)


@pytest.mark.gpu
def test_resample_arb_batch_over_2e31_samples(dsp, big):
    # the arbitrary-rate batch on a Float32 matrix of odd columns, with a dyadic delta: exact against the closed form
    import test_resample_arb_batched as arb
    from dspb200 import device
    torch = big.torch
    x, n_el = big.typed(F32)
    nphi, hlen, W = 32, 32 * 8 - 3, 64
    delta = nphi * 0.75                                  # outputs 4 apart advance 3 whole samples
    ldx = (1 << 24) + 1
    ncols = n_el // ldx
    n0 = 3
    assert ldx * ncols > E31
    h = rk.int_taps(np.random.default_rng(54), hlen, F32)
    plan = dsp._lib.ResampleArbPlan(F32, h, nphi)
    tpp = -(-hlen // nphi)
    nout = (ldx - n0 - 1) * 4 // 3 - 8
    out = _alloc(torch, nout * ncols, plan.out_dtype)
    try:
        plan.exec_batch_dev(x.data_ptr(), ldx, ldx, ncols, n0, 0.0, delta, out.data_ptr(), nout, 0)
        device.sync()
        for c, i in col_probes(ldx, ncols, 4, W):
            j = min(max(0, (i - n0) * 4 // 3), nout - W) // 4 * 4
            q = j * 3 // 4
            a = max(0, n0 + q - (tpp - 1))
            b = min(ldx, n0 + ((j + W - 1) * 3) // 4 + 1)
            xw = _host(x, c * ldx + a, c * ldx + b).reshape(-1, 1)
            want = arb.closed_form(xw, b - a, h, nphi, n0 + q - a, delta, W, plan.out_dtype)[:, 0]
            assert np.array_equal(_host(out, c * nout + j, c * nout + j + W), want), (c, j)
    finally:
        del out
        _free(torch, plan)


@pytest.mark.gpu
@pytest.mark.parametrize("length", MATRIX_LENS, ids=["odd", "aligned"])
def test_welch_batch_and_stream_channels_over_2e31(dsp, big, length):
    # every checked channel against the float64 reference; the streaming accumulation of the whole matrix then its power
    # equals the batched call bit for bit (dspb200.h)
    torch = big.torch
    from dspb200 import device
    x, n_el = big.typed(F32)
    n = N = 4096
    hop = 2048
    nchan = n_el // length
    assert length * nchan > E31
    w = kp.window_of("hann", n, None)
    plan = kp._plan(dsp, F32, n, hop, N, True, w)
    k = plan.nsegments(length)
    r = k * kp.norm2_of(w, n)
    nout = plan.nout
    out = _alloc(torch, nout * nchan, F32)
    acc = _alloc(torch, nout * nchan, torch.float64)
    hist = _alloc(torch, n * nchan, F32)
    out2 = _alloc(torch, nout * nchan, F32)
    try:
        plan.welch_batch_dev(x.data_ptr(), length, nchan, r, out.data_ptr(), 0)
        plan.welch_stream_dev(None, 0, hist.data_ptr(), n, x.data_ptr(), length, nchan, k, acc.data_ptr(), 0, 0)
        plan.welch_stream_power_dev(acc.data_ptr(), nchan, r, out2.data_ptr(), 0)
        device.sync()
        assert torch.equal(out, out2)
        for c in limit_cols(length, nchan, 4):
            X, en = kp.ref_segments(_host(x, c * length, (c + 1) * length), n, hop, N, w)
            kp.check_welch(_host(out, c * nout, (c + 1) * nout), X, en, N, True, r, kp.eps(F32), k, c)
    finally:
        del out, acc, hist, out2
        _free(torch, plan)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4096, 4095], ids=["aligned", "odd"])
def test_mt_pgram_batch_over_2e31(dsp, big, n):
    import test_mt_batched as mt
    from dspb200 import device
    torch = big.torch
    x, n_el = big.typed(F32)
    nchan = n_el // n
    assert n * nchan > E31
    plan = dsp._lib.MtPlan(F32, n, 0, 4096, True, mt.tapers(n, 3))
    nout = plan.nout
    out = _alloc(torch, nout * nchan, F32)
    try:
        plan.mt_pgram_batch_dev(x.data_ptr(), n, nchan, out.data_ptr(), 0)
        vec = device.DeviceArray((nout,), F32)
        for c in limit_cols(n, nchan, 4):
            plan.mt_pgram_dev(x.data_ptr() + 4 * c * n, n, vec.ptr, 0)
            assert kp.same_bits(vec.to_host(), _host(out, c * nout, (c + 1) * nout)), c
    finally:
        del out
        _free(torch, plan)


@pytest.mark.gpu
@pytest.mark.parametrize("length", MATRIX_LENS, ids=["odd", "aligned"])
def test_mt_spectrogram_batch_over_2e31(dsp, big, length):
    import test_mt_batched as mt
    from dspb200 import device
    torch = big.torch
    x, n_el = big.typed(F32)
    n, hop = 4096, 2048
    nchan = n_el // length
    plan = dsp._lib.MtPlan(F32, n, n - hop, n, True, mt.tapers(n, 3))
    k = plan.nsegments(length)
    per = plan.nout * k
    assert length * nchan > E31
    out = _alloc(torch, per * nchan, F32)
    try:
        plan.mt_spectrogram_batch_dev(x.data_ptr(), length, nchan, out.data_ptr(), 0)
        vec = device.DeviceArray((per,), F32)
        for c in limit_cols(length, nchan, 4):
            plan.mt_spectrogram_dev(x.data_ptr() + 4 * c * length, length, vec.ptr, 0)
            assert kp.same_bits(vec.to_host(), _host(out, c * per, (c + 1) * per)), c
    finally:
        del out
        _free(torch, plan)


@pytest.mark.gpu
@pytest.mark.parametrize("length", MATRIX_LENS, ids=["odd", "aligned"])
@pytest.mark.parametrize("psd", [1, 0], ids=["psd", "raw"])
def test_stft_channels_over_4gib(dsp, big, length, psd):
    # every checked channel of the batched STFT equals the call on that channel's pointer bit for bit; the raw spectra
    # (twice the input's bytes) run over the first 4 GiB + 2 channels of the buffer
    from dspb200 import device
    torch = big.torch
    x, n_el = big.typed(F32)
    n, hop = 4096, 2048
    nchan = n_el // length if psd else B32 // 4 // length + 2
    assert length * nchan * 4 > B32 and (not psd or length * nchan > E31)
    w = kp.window_of("hann", n, None)
    plan = kp._plan(dsp, F32, n, hop, n, True, w)
    r = kp.norm2_of(w, n)
    k = plan.nsegments(length)
    per = plan.nout * k
    odt = F32 if psd else C64
    out = _alloc(torch, per * nchan, odt)
    try:
        plan.stft_dev(x.data_ptr(), length, nchan, r, psd, out.data_ptr(), 0)
        vec = device.DeviceArray((per,), odt)
        for c in limit_cols(length, nchan, 4):
            plan.stft_dev(x.data_ptr() + 4 * c * length, length, 1, r, psd, vec.ptr, 0)
            assert kp.same_bits(vec.to_host(), _host(out, c * per, (c + 1) * per)), c
    finally:
        del out
        _free(torch, plan)


@pytest.mark.gpu
def test_stft_long_column_pairs(dsp, big):
    # the PSD columns of one 2^31 + 2^21 + 3 sample column: columns 2u and 2u+1 equal the two-segment call at 2u*hop
    from dspb200 import device
    torch = big.torch
    x, nx = big.typed(F32)
    n, hop = 4096, 2048
    w = kp.window_of("hann", n, None)
    plan = kp._plan(dsp, F32, n, hop, n, True, w)
    r = kp.norm2_of(w, n)
    k = plan.nsegments(nx)
    nout = plan.nout
    out = _alloc(torch, nout * k, F32)
    try:
        plan.stft_dev(x.data_ptr(), nx, 1, r, 1, out.data_ptr(), 0)
        tw = device.DeviceArray((2 * nout,), F32)
        us = {0, (k - 2) // 2} | {max(0, e // (2 * hop) + d) for e in (E31, B32 // 4) for d in (-1, 0)}
        for u in sorted(us):
            assert 2 * u + 1 < k
            plan.stft_dev(x.data_ptr() + 4 * 2 * u * hop, hop + n, 1, r, 1, tw.ptr, 0)
            assert kp.same_bits(tw.to_host(), _host(out, 2 * u * nout, (2 * u + 2) * nout)), u
        assert any(2 * u * hop < E31 <= (2 * u + 1) * hop + n for u in us)
    finally:
        del out
        _free(torch, plan)


# =============================================================================== GPU, C: host pointers over 4 GiB

@pytest.mark.gpu
def test_host_pointer_paths_over_4gib(dsp, big):
    # the chunked host paths (fftfilt, welch_pgram, resample) on a pageable Float32 array of more than 2^31 samples
    import os
    from dspb200 import device
    torch = big.torch
    xd, nx = big.typed(F32)
    need = 2 * nx * 4 + (nx // 4 + (1 << 20)) * 4
    avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if avail < need + (4 << 30):
        pytest.skip(f"needs {need} bytes of free host memory ({avail} free)")
    x = xd.cpu().numpy()
    assert x.size > E31 and x.nbytes > B32
    W = 64
    rng = np.random.default_rng(55)
    # fftfilt
    nv = 4097
    v = int_taps(rng, nv, F32)
    plan = dsp._lib.OsPlan(v, 16384)
    y = np.empty(nx, F32)
    try:
        plan.exec(x, y, nx, 1, nx)
        for i in probe_starts(nx, W, 4, seed=55):
            a = max(0, i - (nv - 1))
            check_exact(y[i:i + W], exact_conv(x[a:i + W], v)[i - a:i - a + W], False, what=("fftfilt", i))
    finally:
        del y
        plan.close()
    # welch_pgram against the device call on the same samples, within the bound at m = all segments
    n, hop = 4096, 2048
    spec = kp._plan(dsp, F32, n, hop, n, True, None)
    try:
        k = spec.nsegments(nx)
        r = float(k * n)
        ph = np.empty(spec.nout, F32)
        spec.welch(x, r, ph)
        pd = device.DeviceArray((spec.nout,), F32)
        spec.welch_dev(xd.data_ptr(), nx, r, pd.ptr, 0)
        pd = pd.to_host().astype(np.float64)
        mult = kp.bins_and_mult(n, True)[1]
        S = pd * r / k / mult
        err = np.abs(ph.astype(np.float64) * r / k / mult - S)
        assert np.all(err <= 2 * power_bound(S, n * 64.0, kp.eps(F32), n, k))
    finally:
        spec.close()
    # decimating resample, exact at probes
    I, D, hlen = 1, 4, 40
    h = rk.int_taps(rng, hlen, F32)
    rs = dsp._lib.ResamplePlan(F32, h, I, D)
    try:
        nout = -(-nx // D)
        n0, phi0 = 5, 0
        out = np.empty(nout, F32)
        rs.exec(x, nx, 1, n0, phi0, out, nout)
        for j in probe_starts(nout, W, 4, seed=56, extra=[(E31 - n0) // D - W // 2, (B32 // 4 - n0) // D - W // 2]):
            want = rs_probe_want(lambda a, b: x[a:b], nx, h, I, D, n0, phi0, j, W)
            assert np.array_equal(out[j:j + W], want), j
    finally:
        rs.close()
        del x
        _free(torch)
