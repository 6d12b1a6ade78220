"""Every kernel path of the rational polyphase resampler (csrc/resample.cu) against a direct polyphase sum.

`rs_launch` sends a call to one of four kernel families, each compiled as several instances: the pipelined multi-phase
kernel (mp2), the multi-phase kernel (mp), the register-tiled kernel and the generic one-output-per-thread kernel.
`expected_family` restates that routing, so the case table can show that every family and every mp / mp2 instance is
reached, on both sides of each size limit.

The main check is exact.  Taps are integers in [-4, 4] and samples integers in [-8, 8] (both parts for complex input),
so every product and partial sum is exact in Float32 (|sum| <= 32 * taps per phase, far below 2^24).  Each output must
then equal the float64 reference bit for bit, whatever the kernel, type or accumulation order.  A wrong tap row or a
one-sample shift at a few tile or CTA boundaries fails that; a norm-relative bound over 10^6 outputs may not notice it.

The CPU tests check the reference itself and the coverage of the case table; the rest need a GPU."""
import math
from fractions import Fraction

import numpy as np
import pytest

from conftest import relerr
from oracle import filters as of

F32, F64, C64, C128 = (np.dtype(t) for t in (np.float32, np.float64, np.complex64, np.complex128))
# the six (input, taps) combinations that select distinct (input, tap, output) instances in rs_run (resample.cu:671-679);
# Float64 input with Float32 taps and ComplexF64 input with Float32 taps share the Float64-tap instances
TRIPLES = ((F32, F32), (F32, F64), (F64, F64), (C64, F32), (C64, F64), (C128, F64))
MP_RATES = ((2, 1), (2, 3), (3, 1), (3, 2), (3, 4), (4, 1), (4, 3))  # the switches in rs_launch (resample.cu:619-639)
SMEM_OPTIN = 227 * 1024          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
H100_SMS = 132
MAX_CTAS_PER_SM = 2048 // 256    # thread limit of an SM: no more 256-thread mp2 CTAs than this can be resident


# =============================================================================== reference

def polyphase_ref(x, h, I, D, n0, phi0, nout):
    """y[j] = sum_t h[phi + t*I] * x[n - t] with p = phi0 + j*D, n = n0 + p // I, phi = p % I; samples outside the
    stored range are zero.  x is a vector or an (nx, ncols) array of columns.  Float64 / complex128 arithmetic."""
    x = np.asarray(x)
    xs = x.astype(np.complex128 if np.iscomplexobj(x) else np.float64).reshape(x.shape[0], -1)
    nx, ncols = xs.shape
    h = np.asarray(h, dtype=np.float64)
    tpp = -(-h.size // I)
    hp = np.zeros(tpp * I)
    hp[:h.size] = h
    # xpad[s + tpp - 1] = x[s] for s in [-(tpp - 1), nx + tpp - 1]: zero outside the stored range
    xpad = np.concatenate([np.zeros((tpp - 1, ncols)), xs, np.zeros((tpp, ncols))]).astype(xs.dtype)
    p = phi0 + np.arange(nout, dtype=np.int64) * D
    phi = p % I
    # a window whose newest sample is past nx + tpp - 1 reads only zeros, as it does from there
    base = np.minimum(n0 + p // I, nx + tpp - 1) + (tpp - 1)
    y = np.zeros((nout, ncols), dtype=xs.dtype)
    for t in range(tpp):
        y += hp[phi + t * I][:, None] * xpad[base - t]
    return y.reshape(nout) if x.ndim == 1 else y


def int_taps(rng, hlen, dt):
    return rng.integers(-4, 5, hlen).astype(dt)


def int_signal(rng, shape, dt):
    dt = np.dtype(dt)
    v = rng.integers(-8, 9, shape).astype(np.float64)
    if dt.kind == "c":
        v = v + 1j * rng.integers(-8, 9, shape)
    return v.astype(dt)


def _resample_phase(hlen, I):
    """undelay! of a fresh filter: the (n0, phi0) that resample() starts from, rounded from the same floating-point
    expression as filters.resample_phase and the oracle."""
    if I == 1:
        return int(np.round((hlen - 1) / 2)), 0
    return divmod(int(np.round((hlen - 1) / (2 * I) * I)), I)


# =============================================================================== routing restated from rs_launch

def _sizes(dtype_x, dtype_h):
    """Byte sizes (EX, TR, EO) of the instance rs_run picks (resample.cu:671-679; output type :735-736)."""
    x = np.dtype(dtype_x)
    tr = 8 if x in (F64, C128) or np.dtype(dtype_h) == F64 else 4
    return x.itemsize, tr, tr * (2 if x.kind == "c" else 1)


def mp_g(dtype_x, dtype_h):
    """G of the mp / mp2 instances: 4 for Float32 arithmetic, 2 for Float64 (resample.cu:617)."""
    return 4 if _sizes(dtype_x, dtype_h)[1] == 4 else 2


def mp2_v3(I, D, dtype_x, dtype_h):
    """rs_v3 (resample.cu:274-278): True where mp2 stages the taps in shared memory, False for constant-bank taps."""
    eo = _sizes(dtype_x, dtype_h)[2]
    G = mp_g(dtype_x, dtype_h)
    NO, GD = I * G, G * D
    est = (((NO - 1) * D) // I + 8 + NO) * (eo // 4) + I * 4
    return est <= 80 and 8 % GD == 0


def _mp_smem(I, D, tpp8, dtype_x, dtype_h, pipelined):
    """Dynamic shared memory of rs_launch_mp2 (resample.cu:576-579) or rs_launch_mp (:542-545); rs_mp at :176-186."""
    ex, tr, eo = _sizes(dtype_x, dtype_h)
    G = mp_g(dtype_x, dtype_h)
    NO, GD = I * G, G * D
    SK, SKO = int(GD % 2 == 0), int(NO % 2 == 0)
    xtile_len = 255 * GD + ((NO - 1) * D) // I + tpp8 + 1
    xpos_end = xtile_len + SK * (xtile_len // GD)
    obytes = (256 * NO + SKO * 256 + 2) * eo                       # opos(TILE_OUT) + 2 outputs
    if pipelined:
        xbuf_elems = (xpos_end + 3) & ~1
        return 2 * xbuf_elems * ex + obytes + 16 + (I * 64 * tr if mp2_v3(I, D, dtype_x, dtype_h) else 0)
    return I * tpp8 * tr + max((xpos_end + 2) * ex, obytes) + 16


def tiled_g(D, dtype_x, dtype_h):
    """G of resample_tiled_kernel<D, G> (resample.cu:648-651)."""
    f32 = _sizes(dtype_x, dtype_h)[1] == 4
    return {1: (7, 3), 2: (7, 3), 3: (5, 3), 4: (4, 2)}[D][0 if f32 else 1]


def _tiled_smem(I, D, tpp8, dtype_x, dtype_h):
    """Dynamic shared memory of rs_launch_tiled (resample.cu:513-521)."""
    ex, tr, eo = _sizes(dtype_x, dtype_h)
    G = tiled_g(D, dtype_x, dtype_h)
    tile_out = I * G * (256 // I)
    span = ((tile_out - 1) * D) // I + tpp8 + (G - 1) * D + 16
    return I * tpp8 * tr + max((span + 2) * ex, tile_out * eo) + 16


def expected_family(I, D, hlen, dtype_x, dtype_h, ncols=1):
    """The kernel family rs_launch (resample.cu:613-669) runs for a plan of rate I//D with hlen taps."""
    tpp = -(-hlen // I)
    tpp8 = -(-tpp // 8) * 8
    if (I, D) in MP_RATES:                                                                   # :614, :619-639
        if tpp8 <= 64 and _mp_smem(I, D, tpp8, dtype_x, dtype_h, True) <= min(SMEM_OPTIN, 72 * 1024):   # :571, :580
            return "mp2"                                                 # 1-D persistent grid: any number of columns
        if (tpp8 <= 512 and _mp_smem(I, D, tpp8, dtype_x, dtype_h, False) <= min(SMEM_OPTIN, 200 * 1024)
                and ncols <= 65535):                                                         # :546-548
            return "mp"
    if I <= 128 and D <= 4:                                                                  # :642
        if _tiled_smem(I, D, tpp8, dtype_x, dtype_h) <= min(SMEM_OPTIN, 160 * 1024) and ncols <= 65535:  # :522-525
            return "tiled"
    return "generic"                                                                         # :655-668


def tile_outputs(family, I, D, dtype_x, dtype_h):
    """Outputs per tile (CTA work item) of the family."""
    if family in ("mp", "mp2"):
        return 256 * I * mp_g(dtype_x, dtype_h)                                              # rs_mp::TILE_OUT
    if family == "tiled":
        return I * tiled_g(D, dtype_x, dtype_h) * (256 // I)                                 # :513-516
    return 256                                                                               # RS_NT


def _tiled_tpp_limit(I, D, dtype_x, dtype_h):
    """Largest taps per phase the tiled kernel takes (a multiple of 8: its bank rows are padded to one)."""
    tpp8 = 8
    while _tiled_smem(I, D, tpp8 + 8, dtype_x, dtype_h) <= min(SMEM_OPTIN, 160 * 1024):
        tpp8 += 8
    return tpp8


# =============================================================================== case table

def _build_cases():
    cases = []
    for I, D in MP_RATES:                      # 13 taps per phase: one full 8-tap chunk, then a partial one
        for tx, th in TRIPLES:
            cases.append((I, D, 13 * I - 1, tx, th))
    for k, (I, D) in enumerate(MP_RATES):      # tpp 64 (largest mp2 bank) against 65 (mp)
        tx, th = TRIPLES[k % len(TRIPLES)]
        cases += [(I, D, 64 * I, tx, th), (I, D, 64 * I + 1, tx, th)]
    cases += [(3, 2, 56 * 3, C128, F64), (3, 2, 57 * 3, C128, F64)]       # mp2's 72 KB cap: tpp 56 (mp2), 57 (mp)
    cases += [(2, 1, 512 * 2, F32, F32), (2, 1, 512 * 2 + 1, F32, F32)]     # tpp8 512 (mp) against 520 (tiled)
    tiled_and_generic = ((1, 1), (5, 1), (1, 2), (5, 2), (7, 3), (1, 3), (9, 4), (1, 4), (128, 1), (128, 3),
                         (129, 1), (129, 4), (11, 5), (3, 7), (1, 5))
    for k, (I, D) in enumerate(tiled_and_generic):
        tx, th = TRIPLES[k % len(TRIPLES)]
        cases.append((I, D, 10 * I + 1, tx, th))                           # 11 taps per phase
    for I, D, tx, th in ((128, 1, F32, F32), (5, 2, F64, F64)):           # the tiled kernel's shared-memory limit
        lim = _tiled_tpp_limit(I, D, tx, th)
        cases += [(I, D, lim * I, tx, th), (I, D, lim * I + 1, tx, th)]
    return cases


CASES = _build_cases()
# for the phase, range and streaming tests: every mp2 rate, every mp rate (tpp 65), then tiled rates and a generic one
PHASE_CASES = ([(I, D, 13 * I - 1) + TRIPLES[k % 6] for k, (I, D) in enumerate(MP_RATES)]
               + [(I, D, 64 * I + 1) + TRIPLES[(k + 3) % 6] for k, (I, D) in enumerate(MP_RATES)]
               + [(5, 2, 51, C64, F32), (7, 3, 60, F32, F32), (9, 4, 100, C128, F64), (11, 5, 40, F64, F64)])


def _case_id(c):
    I, D, hlen, tx, th = c
    return f"{I}/{D}-{tx.name}-{th.name}-h{hlen}-{expected_family(I, D, hlen, tx, th)}"


# =============================================================================== CPU: the reference and the table

@pytest.mark.parametrize("rate", ["1/1", "2/1", "1/3", "3/2", "4/3", "5/7", "13/4"])
def test_polyphase_ref_matches_oracle_resample(rate):
    r = Fraction(rate)
    I, D = r.numerator, r.denominator
    rng = np.random.default_rng(11)
    for hlen, nx, dt in ((1, 9, F64), (7, 40, F64), (29, 113, C128), (64, 5, F64)):
        h = int_taps(rng, hlen, F64)
        x = int_signal(rng, nx, dt)
        n0, phi0 = _resample_phase(hlen, I)
        nout = math.ceil(nx * r)
        want = polyphase_ref(x, h, I, D, n0, phi0, nout)
        assert np.array_equal(of.resample(x, r, h, f64=True), want), (rate, hlen)
        if r != 1:          # the literal single-rate loop (stream_filt.jl:409-428) does not consume the undelay
            assert np.array_equal(of.resample_literal(x, r, h), want), (rate, hlen)
        xm = np.stack([x, x[::-1], 2 * x], axis=1)
        ym = polyphase_ref(xm, h, I, D, n0, phi0, nout)
        assert np.array_equal(ym[:, 0], want) and np.array_equal(ym[:, 2], 2 * want)
        assert np.array_equal(ym[:, 1], polyphase_ref(x[::-1], h, I, D, n0, phi0, nout))


@pytest.mark.parametrize("rate", ["2/1", "3/2", "4/3", "1/3", "7/3"])
def test_polyphase_ref_matches_fir_filter_state(rate):
    # a FIRFilter starts at n0 = 0, phi0 = 0 with zero history; setphase moves both; chunks carry the state
    r = Fraction(rate)
    I, D = r.numerator, r.denominator
    rng = np.random.default_rng(12)
    h = int_taps(rng, 5 * I + 2, F64)
    x = int_signal(rng, 300, F64)
    sf = of.FIRFilterState(h, r)
    y = sf.filt(x)
    assert np.array_equal(y, polyphase_ref(x, h, I, D, 0, 0, y.size))
    for tau in (0.4, 1.7, 3.0):
        sf = of.FIRFilterState(h, r)
        sf.setphase(tau)
        n0, phi0 = sf.input_deficit - 1, (sf.phi_idx - 1 if I > 1 else 0)
        parts = [sf.filt(x[a:b]) for a, b in ((0, 1), (1, 3), (3, 50), (50, 300))]
        y = np.concatenate(parts)
        assert np.array_equal(y, polyphase_ref(x, h, I, D, n0, phi0, y.size)), (rate, tau)


def test_case_table_covers_every_kernel_family():
    fam = {c: expected_family(*c) for c in CASES}
    got = {f: [c for c in CASES if fam[c] == f] for f in ("mp2", "mp", "tiled", "generic")}
    for I, D in MP_RATES:
        for tx, th in TRIPLES:
            if _mp_smem(I, D, 8, tx, th, True) <= 72 * 1024:          # instance reachable at all
                assert any(c[:2] == (I, D) and c[3:] == (tx, th) for c in got["mp2"]), (I, D, tx, th)
            else:                                                      # over the 72 KB cap at any bank size
                assert any(c[:2] == (I, D) and c[3:] == (tx, th) for c in got["mp"]), (I, D, tx, th)
        assert any(c[:2] == (I, D) for c in got["mp"]), (I, D)
    # both mp2 tap sources and both mp2 chunk loops (tpp = 13: full + partial chunk) are exercised
    assert {mp2_v3(I, D, tx, th) for I, D, _, tx, th in got["mp2"]} == {True, False}
    assert {c[1] for c in got["tiled"]} == {1, 2, 3, 4}
    assert any(c[0] == 128 for c in got["tiled"]) and any(c[0] == 129 for c in got["generic"])
    assert any(c[1] >= 5 for c in got["generic"])
    # generic with the bank in shared memory and with the bank read from global memory (resample.cu:659-661)
    bank = [c[0] * -(-c[2] // c[0]) * _sizes(c[3], c[4])[1] for c in got["generic"]]
    assert min(bank) <= 96 * 1024 < max(bank)
    # size limits, both sides: mp2 at tpp 64 / mp at 65; mp at tpp8 512 / tiled past it; tiled shared memory
    for I, D in MP_RATES:
        (lo,) = [c for c in CASES if c[:3] == (I, D, 64 * I)]
        hi = (I, D, 64 * I + 1) + lo[3:]
        assert fam[lo] == "mp2" and fam[hi] == "mp", (I, D)
    assert fam[(3, 2, 168, C128, F64)] == "mp2" and fam[(3, 2, 171, C128, F64)] == "mp"
    assert fam[(2, 1, 1024, F32, F32)] == "mp" and fam[(2, 1, 1025, F32, F32)] == "tiled"
    for I, D, tx, th in ((128, 1, F32, F32), (5, 2, F64, F64)):
        lim = _tiled_tpp_limit(I, D, tx, th)
        assert fam[(I, D, lim * I, tx, th)] == "tiled" and fam[(I, D, lim * I + 1, tx, th)] == "generic"
    # mp's own 200 KB shared-memory cap never binds below its tpp8 <= 512 limit, so that limit is the boundary
    assert max(_mp_smem(I, D, 512, tx, th, False) for I, D in MP_RATES for tx, th in TRIPLES) < 200 * 1024
    # the ComplexF32 / ComplexF64 4//3 instances stay over mp2's 72 KB even with 8 taps per phase
    assert expected_family(4, 3, 7, C64, F32) == "mp" and expected_family(4, 3, 7, C128, F64) == "mp"
    # the phase, range and streaming tests run every mp2 and mp rate, a tiled rate with D > 1 and a generic rate
    phase = [(c[:2], expected_family(*c)) for c in PHASE_CASES]
    assert {(r, f) for r in MP_RATES for f in ("mp2", "mp")} <= set(phase)
    assert phase[-4][1] == "tiled" and phase[-4][0][1] > 1 and phase[-1][1] == "generic"
    # more than 65535 columns: mp2 keeps them (one-dimensional grid), mp and tiled hand them to the generic kernel
    assert expected_family(3, 2, 38, F32, F32, 70000) == "mp2"
    assert expected_family(3, 2, 3 * 65, F32, F32, 70000) == "generic"
    assert expected_family(5, 2, 51, F32, F32, 70000) == "generic"


# =============================================================================== GPU

@pytest.fixture(scope="module")
def dsp():
    return pytest.importorskip("dspb200")


def _plan_exec(dsp, plan, x, n0, phi0, nout):
    """plan.exec on an (nx,) or (nx, ncols) array; returns the output in the plan's output type."""
    xf = np.asfortranarray(x.reshape(x.shape[0], -1))
    out = np.empty((nout, xf.shape[1]), dtype=plan.out_dtype, order="F")
    plan.exec(xf, xf.shape[0], xf.shape[1], n0, phi0, out, nout)
    return out.reshape(nout) if x.ndim == 1 else out


@pytest.mark.gpu
@pytest.mark.parametrize("I,D,hlen,tx,th", CASES, ids=[_case_id(c) for c in CASES])
def test_exact_at_tile_and_signal_edges(dsp, I, D, hlen, tx, th):
    fam = expected_family(I, D, hlen, tx, th)
    tpp = -(-hlen // I)
    T = tile_outputs(fam, I, D, tx, th)
    rng = np.random.default_rng([I, D, hlen, tx.num, th.num])
    h = int_taps(rng, hlen, th)
    n0, phi0 = _resample_phase(hlen, I)
    plan = dsp._lib.ResamplePlan(tx, h, I, D)
    try:
        shapes = [(nx, math.ceil((nx + tpp) * I / D) + 2, 1) for nx in sorted({1, 2, max(tpp - 1, 1), tpp})]
        shapes += [(math.ceil(nout * D / I) + 1, nout, 1) for nout in (T - 1, T, T + 1)]
        shapes += [(math.ceil((2 * T + 5) * D / I), 2 * T + 5, 3), (math.ceil((T + 37) * D / I), T + 37, 70)]
        for nx, nout, ncols in shapes:
            x = int_signal(rng, (nx, ncols) if ncols > 1 else nx, tx)
            y = _plan_exec(dsp, plan, x, n0, phi0, nout)
            assert np.array_equal(y, polyphase_ref(x, h, I, D, n0, phi0, nout)), (fam, nx, nout, ncols)
    finally:
        plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("tx,th", [(F32, F32), (F64, F64)], ids=["f32", "f64"])
@pytest.mark.parametrize("I,D", MP_RATES, ids=[f"{i}/{d}" for i, d in MP_RATES])
def test_exact_mp2_persistent_ctas_run_several_tiles(dsp, I, D, tx, th):
    # enough tiles that every persistent CTA (at most 132 SMs x 8 resident) runs at least three, so the double-buffered
    # tile loads, the buffer flip and the copy-out of later tiles all run
    hlen = 9 * I - 1
    assert expected_family(I, D, hlen, tx, th) == "mp2"
    T = tile_outputs("mp2", I, D, tx, th)
    nout = 3 * H100_SMS * MAX_CTAS_PER_SM * T + 2 * T // 3
    nx = math.ceil(nout * D / I)
    rng = np.random.default_rng([I, D, tx.num])
    h = int_taps(rng, hlen, th)
    x = int_signal(rng, nx, tx)
    plan = dsp._lib.ResamplePlan(tx, h, I, D)
    try:
        n0, phi0 = 4, I - 1
        y = _plan_exec(dsp, plan, x, n0, phi0, nout)
        bad = np.flatnonzero(y != polyphase_ref(x, h, I, D, n0, phi0, nout))
        assert bad.size == 0, (bad.size, bad[:8])
    finally:
        plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("I,D,hlen,tx,th", PHASE_CASES, ids=[_case_id(c) for c in PHASE_CASES])
def test_exec_dev_every_phase_and_offset(dsp, I, D, hlen, tx, th):
    # the mp / mp2 tile origin jA follows phi0; n0 past the end of the signal leaves only the tail of the windows
    from dspb200 import device
    fam = expected_family(I, D, hlen, tx, th)
    tpp = -(-hlen // I)
    T = tile_outputs(fam, I, D, tx, th)
    nout = 2 * T + 3
    nx = math.ceil(nout * D / I)
    rng = np.random.default_rng([I, D, hlen])
    h = int_taps(rng, hlen, th)
    x = int_signal(rng, nx, tx)
    plan = dsp._lib.ResamplePlan(tx, h, I, D)
    try:
        dx = device.to_device(x)
        out = device.DeviceArray((nout,), plan.out_dtype)
        for phi0 in range(I):
            for n0 in (0, 1, tpp - 1, tpp + 5, nx - 2, nx + 3):
                plan.exec_dev(dx.ptr, nx, 1, n0, phi0, out.ptr, nout, 0)
                device.sync()
                assert np.array_equal(out.to_host(), polyphase_ref(x, h, I, D, n0, phi0, nout)), (fam, phi0, n0)
    finally:
        plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("I,D,hlen,tx,th", PHASE_CASES, ids=[_case_id(c) for c in PHASE_CASES])
def test_exec_range_dev_unaligned_ranges_reassemble(dsp, I, D, hlen, tx, th):
    # 8 output ranges cut off the tile grid (1-sample ranges, ranges inside one tile, ranges across several), each
    # given only the input samples it reads, at their global offsets
    from dspb200 import device
    fam = expected_family(I, D, hlen, tx, th)
    tpp = -(-hlen // I)
    T = tile_outputs(fam, I, D, tx, th)
    nout = 3 * T + 11
    nx = math.ceil(nout * D / I)
    n0, phi0 = 2, I - 1
    rng = np.random.default_rng([I, D, hlen, 1])
    h = int_taps(rng, hlen, th)
    x = int_signal(rng, nx, tx)
    cuts = [0, 1, 3, T - 1, T + 2, T + 3 + T // 2, 2 * T + 1, nout - 1, nout]
    plan = dsp._lib.ResamplePlan(tx, h, I, D)
    try:
        whole = device.DeviceArray((nout,), plan.out_dtype)
        plan.exec_dev(device.to_device(x).ptr, nx, 1, n0, phi0, whole.ptr, nout, 0)
        device.sync()
        whole = whole.to_host()
        got = np.empty_like(whole)
        for b, e in zip(cuts[:-1], cuts[1:]):
            lo = max(0, n0 + (phi0 + b * D) // I - (tpp - 1))
            hi = max(lo, min(nx, n0 + (phi0 + (e - 1) * D) // I + 1))
            local = device.to_device(x[lo:hi])
            part = device.DeviceArray((e - b,), plan.out_dtype)
            plan.exec_range_dev(local.ptr, lo, hi - lo, n0, phi0, part.ptr, b, e - b, 0)
            device.sync()
            got[b:e] = part.to_host()
        assert np.array_equal(got, whole), fam
        assert np.array_equal(whole, polyphase_ref(x, h, I, D, n0, phi0, nout)), fam
    finally:
        plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("I,D,hlen,tx,th", PHASE_CASES[:-3], ids=[_case_id(c) for c in PHASE_CASES[:-3]])
def test_fir_filter_chunks_carry_phase_and_deficit(dsp, I, D, hlen, tx, th):
    # streaming is the caller that passes a new phi0 / n0 on every call: chunks of 1, 2, 3, a tile of input - 1,
    # a tile + 1 and the rest equal one call, the reference's stateful loops and the direct sum
    fam = expected_family(I, D, hlen, tx, th)
    T_in = tile_outputs(fam, I, D, tx, th) * D // I
    chunks = (1, 2, 3, T_in - 1, T_in + 1, T_in + 5)
    rng = np.random.default_rng([I, D, hlen, 2])
    h = int_taps(rng, hlen, th)
    x = int_signal(rng, sum(chunks), tx)
    whole = dsp.FIRFilter(h, Fraction(I, D)).filt(x)
    assert np.array_equal(whole, polyphase_ref(x, h, I, D, 0, 0, whole.size)), fam
    f, ref = dsp.FIRFilter(h, Fraction(I, D)), of.FIRFilterState(h, Fraction(I, D))
    parts, pos = [], 0
    for n in chunks:
        part = f.filt(x[pos:pos + n])
        want = ref.filt(x[pos:pos + n])
        assert part.dtype == whole.dtype and np.array_equal(part, want), (fam, pos, n)
        assert (f.phi_idx, f.input_deficit) == (ref.phi_idx, ref.input_deficit), (fam, pos, n)
        parts.append(part)
        pos += n
    assert np.array_equal(np.concatenate(parts), whole), fam


@pytest.mark.gpu
@pytest.mark.parametrize("I,D,hlen", [(3, 2, 38), (3, 2, 3 * 65), (5, 2, 51)], ids=["mp2", "mp", "tiled"])
def test_resample_70000_columns(dsp, I, D, hlen):
    # more columns than gridDim.y holds: mp2 runs them on its one-dimensional grid, mp and tiled give way to the
    # generic kernel
    ncols, nx = 70000, 5
    fam = expected_family(I, D, hlen, F32, F32, ncols)
    rng = np.random.default_rng([I, D, hlen, 3])
    h = int_taps(rng, hlen, F32)
    x = int_signal(rng, (nx, ncols), F32)
    y = dsp.resample(x, Fraction(I, D), h, dims=0)
    n0, phi0 = _resample_phase(hlen, I)
    nout = math.ceil(nx * I / D)
    assert y.shape == (nout, ncols) and y.dtype == F32
    assert np.array_equal(y, polyphase_ref(x, h, I, D, n0, phi0, nout)), fam


PRECISION_CASES = [("3/2", None, 200_000), ("4/3", None, 200_000), ("5/2", None, 200_000), ("11/5", None, 200_000),
                   ("3/2", 64 * 3 * 2 + 5, 20_000), ("4/1", 64 * 4 + 9, 20_000), ("5/2", 64 * 5 * 2 + 5, 20_000)]


@pytest.mark.gpu
@pytest.mark.parametrize("tx,th", [(F32, F32), (C64, F32), (F64, F64), (C128, F64)],
                         ids=["f32", "c64", "f64", "c128"])
@pytest.mark.parametrize("rate,hlen,nx", PRECISION_CASES, ids=[f"{r}-h{h or 'default'}" for r, h, _ in PRECISION_CASES])
def test_precision_random_data(dsp, rate, hlen, nx, tx, th):
    # random data: Float32 outputs within twice the error of the reference's own Float32 loop, Float64 within 1e-12
    r = Fraction(rate)
    rng = np.random.default_rng([r.numerator, r.denominator, hlen or 0, tx.num])
    h = dsp.resample_filter(r) if hlen is None else rng.standard_normal(hlen) / math.sqrt(hlen)
    h = h.astype(th)
    x = rng.standard_normal(nx)
    if tx.kind == "c":
        x = x + 1j * rng.standard_normal(nx)
    x = x.astype(tx)
    y = dsp.resample(x, r, h)
    truth = of.resample(x, r, h, f64=True)
    assert y.shape == truth.shape
    if y.dtype in (F32, C64):
        assert relerr(y, truth) <= max(2 * relerr(of.resample(x, r, h), truth), 1e-6)
    else:
        assert relerr(y, truth) < 1e-12
