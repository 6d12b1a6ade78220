"""Where and when the device-pointer entry points run: caller streams, several plans and threads, CUDA-graph capture.

include/dspb200.h promises that every `*_exec_dev` call is enqueued on the caller's `stream` and returns without
synchronising, that the plan-less and multitaper `_dev` calls return only after their work on that stream has completed,
and that different plans may be used at once ("one caller at a time per plan").  The kernel-path suites check what the
kernels compute, on stream 0, which serialises with every blocking stream; none of them would notice a launch on stream 0
or on a plan's private stream, a synchronous copy in the middle of a call, a hidden device synchronisation or a stream a
plan keeps from its first call.  This file checks the contract itself.

Every case runs one entry point on a non-blocking torch stream S.  A delay (torch.cuda._sleep, sized from the device clock
to at least 10 times the host time of issuing the call) is queued on S, then the copy of the input from pinned memory;
until that copy lands the input buffer holds sentinels of magnitude 10^6.  The call follows on S, and the output is
copied back on S.  The result must equal the same call on stream 0 bit for bit (the kernel-path suites check that call
against float64 references), so a kernel that does not wait for S reads the sentinels and fails on the first run; nothing
is repeated to catch a race.  Async entry points must leave S busy when they return, the others idle.  The same plan then
runs on a second stream and back; two plans of one entry point run on two streams at once; the async entry points are
captured in CUDA graphs and replayed on new input; four threads run plans and plan-less calls side by side.  The
harness's own checks are shown to fail on planted misuse: a call on stream 0 reads the sentinels, and a stream
synchronisation inside the call fails the asynchrony check.

The case table reaches every `dspb200_*_dev` symbol the header declares, classified from the header's own comments, and
every route whose host code differs (fused and cuFFT spectral sizes, fused and generic overlap-save with and without state,
the four rational resampler families, the single and batched Welch kernels, the warp-per-unit STFT kernel), restated by
the kernel-path suites."""
import ctypes as C
import gc
import os
import re
import threading
import time

import numpy as np
import pytest

from conftest import ROOT
import test_client_kernel_paths as ck
import test_os_kernel_paths as osk
import test_resample_kernel_paths as rk
import test_spectral_kernel_paths as kp
from test_spectral_kernel_paths import F32, F64, C64, Guarded, same_bits

HEADER = os.path.join(ROOT, "include", "dspb200.h")
MIN_DELAY = 0.005            # seconds: the shortest delay queued ahead of a call
DELAY_OVER_WARM = 20         # delay = this many times the host time of a whole warm call (issue, run, copies), at least
ISSUE_RATIO = 10             # the delay must be at least this many times the host time of issuing the call


# =============================================================================== the header's entry points

_TOKEN = re.compile(r"/\*.*?\*/|DSPB200_API\s+[^;{}]*?\b(dspb200_\w+)\s*\(", re.S)
_COMPLETES = re.compile(r"returns?\s+after\s+the\s+work\s+on\s+that\s+stream\s+has\s+completed")


def header_dev_entry_points():
    """{symbol: "sync" | "async"} for every dspb200_*_dev declaration: "sync" when the last comment before it says the
    call returns after the work on its stream has completed, "async" (the conventions block) otherwise."""
    with open(HEADER) as f:
        text = f.read()
    comment, kinds = "", {}
    for m in _TOKEN.finditer(text):
        if m.group(1) is None:
            comment = " ".join(re.sub(r"\n\s*\*(?!/)", " ", m.group(0)).split())
        elif m.group(1).endswith("_dev"):
            kinds[m.group(1)] = "sync" if _COMPLETES.search(comment) else "async"
    return kinds


SYNC_ENTRIES = {"dspb200_conv_nd_exec_dev", "dspb200_conv_nd_os_exec_dev", "dspb200_hilbert_exec_dev",
                "dspb200_periodogram2_exec_dev", "dspb200_mt_pgram_exec_dev", "dspb200_mt_spectrogram_exec_dev",
                "dspb200_mt_pgram_batch_exec_dev", "dspb200_mt_spectrogram_batch_exec_dev",
                "dspb200_mt_cross_spectra_exec_dev"}


# =============================================================================== case table

def _sig(rng, dt, n):
    x = rng.standard_normal(n)
    if np.dtype(dt).kind == "c":
        x = x + 1j * rng.standard_normal(n)
    return x.astype(dt)


class Run:
    """One configured call: input (dtype, count) pairs, output (dtype, count) pairs and call(in_ptrs, out_ptrs, stream).
    `keep` holds the plans; `compare(got, ref, data)` replaces the bitwise comparison."""

    def __init__(self, ins, outs, call, keep=(), compare=None):
        self.ins, self.outs, self.call, self.keep, self.compare = ins, outs, call, keep, compare

    def inputs(self, rng):
        return [_sig(rng, dt, n) for dt, n in self.ins]

    def same(self, got, ref, data):
        if self.compare is not None:
            return self.compare(got, ref, data)
        return all(same_bits(a, b) for a, b in zip(got, ref))


class Case:
    def __init__(self, name, entries, route, build):
        self.name, self.entries, self.route, self.build = name, tuple(entries), route, build

    @property
    def sync(self):
        return self.entries[0] in SYNC_ENTRIES


def _taps_rng(scale):
    return np.random.default_rng(1000 + scale)


# ---- FIR and overlap-save

def _fir(stateful):
    def build(dsp, scale):
        nb, nx, ncols = 33, 5000 * scale + 7, 3
        plan = dsp._lib.FirPlan(_sig(_taps_rng(scale), F32, nb))
        if not stateful:
            return Run([(F32, nx * ncols)], [(F32, nx * ncols)],
                       lambda i, o, st: plan.exec_dev(i[0], nx, ncols, o[0], st), (plan,))
        ns = (nb - 1) * ncols
        return Run([(F32, nx * ncols), (F32, ns)], [(F32, nx * ncols), (F32, ns)],
                   lambda i, o, st: plan.exec_state_dev(i[0], nx, ncols, i[1], o[1], o[0], st), (plan,))
    return build


def _os_route(dt, nv, nfft):
    f64 = dt == F64
    return "fused" if osk.os_fused_ok(nfft or osk.auto_nfft(nv, f64), nv, f64) else "generic"


def _os(dt, nv, nfft, form):
    def build(dsp, scale):
        plan = dsp._lib.OsPlan(_sig(_taps_rng(scale), dt, nv), nfft)
        assert plan.fused == (_os_route(dt, nv, nfft) == "fused")
        assert plan.nfft == (nfft or osk.auto_nfft(nv, dt == F64))
        ncols = 2
        if form == "plain":
            nu = 20000 * scale + 3
            nout = nu + nv - 1
            return Run([(dt, nu * ncols)], [(dt, nout * ncols)],
                       lambda i, o, st: plan.exec_dev(i[0], nu, ncols, o[0], nout, st), (plan,))
        if form == "range":
            nu, cnt = 8000 * scale + 5, 9000 * scale
            return Run([(dt, nu)], [(dt, cnt)], lambda i, o, st: plan.exec_range_dev(i[0], 3000, nu, o[0], 1000, cnt, st),
                       (plan,))
        nx, ns = 30000 * scale + 11, (nv - 1) * ncols
        return Run([(dt, nx * ncols), (dt, ns)], [(dt, nx * ncols), (dt, ns)],
                   lambda i, o, st: plan.exec_state_dev(i[0], nx, ncols, i[1], o[1], o[0], st), (plan,))
    return build


# ---- Welch, STFT, multitaper

def _spec_geometry(nfft, scale):
    n, hop = nfft, nfft // 2
    k = 9 * scale
    return n, hop, k, hop * (k - 1) + n


def _spec_route(dt, nfft):
    return "fused" if kp.fused_size_ok(nfft, dt == F64) else "cufft"


def _spec(dt, nfft, form):
    def build(dsp, scale):
        n, hop, k, length = _spec_geometry(nfft, scale)
        plan = dsp._lib.SpecPlan(dt, n, n - hop, nfft, dt.kind != "c", kp.window_of("hann", n, None))
        assert plan.fused == (_spec_route(dt, nfft) == "fused")
        assert plan.nsegments(length) == k
        nout, re_, r, nchan = plan.nout, kp._real(dt), 1.7, 3
        if form == "welch":
            return Run([(dt, length)], [(re_, nout)], lambda i, o, st: plan.welch_dev(i[0], length, r, o[0], st), (plan,))
        if form == "batch":
            return Run([(dt, length * nchan)], [(re_, nout * nchan)],
                       lambda i, o, st: plan.welch_batch_dev(i[0], length, nchan, r, o[0], st), (plan,))
        if form == "range":
            return Run([(dt, length)], [(re_, nout)],
                       lambda i, o, st: plan.welch_range_dev(i[0], length, 0, 1, k - 1, r, o[0], st), (plan,))
        if form == "triple":
            def call(i, o, st):
                plan.welch_begin_dev(st)
                plan.welch_accumulate_dev(i[0], length, 0, 0, k, st)
                plan.welch_finalize_dev(r, o[0], st)
            return Run([(dt, length)], [(re_, nout)], call, (plan,))
        if form == "stft":
            return Run([(dt, length * nchan)], [(re_, nout * k * nchan)],
                       lambda i, o, st: plan.stft_dev(i[0], length, nchan, r, True, o[0], st), (plan,))
        # streams: a history of n - hop samples, a chunk of nx, every segment that fits
        nhist, ldh, nx = n - hop, n, hop * 5 * scale + 3
        nseg = (nhist + nx - n) // hop + 1
        if form == "stft_stream":
            return Run([(dt, ldh * nchan), (dt, nx * nchan)], [(dt, ldh * nchan), (re_, nout * nseg * nchan)],
                       lambda i, o, st: plan.stft_stream_dev(i[0], nhist, o[0], ldh, i[1], nx, nchan, nseg, r, True, o[1],
                                                             nseg, st), (plan,))
        if form == "welch_stream":
            return Run([(dt, ldh * nchan), (dt, nx * nchan)], [(dt, ldh * nchan), (F64, nout * nchan)],
                       lambda i, o, st: plan.welch_stream_dev(i[0], nhist, o[0], ldh, i[1], nx, nchan, nseg, o[1], False,
                                                              st), (plan,))
        assert form == "welch_stream_power"
        return Run([(F64, nout * nchan)], [(re_, nout * nchan)],
                   lambda i, o, st: plan.welch_stream_power_dev(i[0], nchan, r, o[0], st), (plan,))
    return build


def _stft_route(dt, nfft):
    n, hop, k, length = _spec_geometry(nfft, 1)
    return kp.stft_route(dt, nfft, n, hop, length, 3, True, True)[0] if kp.fused_size_ok(nfft, dt == F64) else "cufft"


def _mt(dt, nfft, form):
    def build(dsp, scale):
        n, hop, k, length = _spec_geometry(nfft, scale)
        tapers = _taps_rng(scale).standard_normal((3, n)) * 0.05
        cross = form == "cross"
        plan = dsp._lib.MtPlan(dt, n, 0 if cross else n - hop, nfft, True, tapers)
        assert plan.fused == (_spec_route(dt, nfft) == "fused")
        nout, re_, nchan = plan.nout, kp._real(dt), 3
        if cross:
            nch, f_lo, nf = 4, 3, 20
            return Run([(dt, nch * n)], [(C64, nch * nch * nf)],
                       lambda i, o, st: plan.cross_spectra_dev(i[0], nch, True, f_lo, nf, False, o[0], st), (plan,))
        if form == "pgram":
            return Run([(dt, n)], [(re_, nout)], lambda i, o, st: plan.mt_pgram_dev(i[0], n, o[0], st), (plan,))
        if form == "spectrogram":
            return Run([(dt, length)], [(re_, nout * k)], lambda i, o, st: plan.mt_spectrogram_dev(i[0], length, o[0], st),
                       (plan,))
        if form == "pgram_batch":
            return Run([(dt, n * nchan)], [(re_, nout * nchan)],
                       lambda i, o, st: plan.mt_pgram_batch_dev(i[0], n, nchan, o[0], st), (plan,))
        assert form == "spectrogram_batch"
        return Run([(dt, length * nchan)], [(re_, nout * k * nchan)],
                   lambda i, o, st: plan.mt_spectrogram_batch_dev(i[0], length, nchan, o[0], st), (plan,))
    return build


# ---- resampling

RS_FAMILIES = {"mp2": (3, 2, 38), "mp": (3, 2, 195), "tiled": (5, 2, 51), "generic": (5, 7, 60)}
ARB_NPHASES, ARB_HLEN, ARB_RATE = 32, 32 * 12, 1.37


def _rs(I, D, hlen, form):
    def build(dsp, scale):
        plan = dsp._lib.ResamplePlan(F32, _sig(_taps_rng(scale), F32, hlen), I, D)
        tpp = -(-hlen // I)
        ncols, nx = 2, 7000 * scale + 13
        n0, phi0 = tpp // 2, 1
        if form == "plain":
            nout = nx * I // D
            return Run([(F32, nx * ncols)], [(F32, nout * ncols)],
                       lambda i, o, st: plan.exec_dev(i[0], nx, ncols, n0, phi0, o[0], nout, st), (plan,))
        if form == "range":
            nloc, cnt = 6000 * scale + 1, 8000 * scale
            return Run([(F32, nloc)], [(F32, cnt)],
                       lambda i, o, st: plan.exec_range_dev(i[0], 500, nloc, n0, phi0, o[0], 300, cnt, st), (plan,))
        assert form == "stream"
        H, nout = tpp - 1, nx * I // D - 1
        return Run([(F32, H * ncols), (F32, nx * ncols)], [(F32, H * ncols), (F32, nout * ncols)],
                   lambda i, o, st: plan.stream_exec_dev(i[0], o[0], i[1], nx, ncols, 1, 0, o[1], nout, nout, st), (plan,))
    return build


def _arb(form):
    def build(dsp, scale):
        plan = dsp._lib.ResampleArbPlan(F32, _sig(_taps_rng(scale), F32, ARB_HLEN), ARB_NPHASES)
        nx, ncols, acc0, delta = 6000 * scale + 9, 3, 0.3, ARB_NPHASES / ARB_RATE
        nout = int(nx * ARB_RATE) - 5
        if form == "plain":
            return Run([(F32, nx)], [(F32, nout)], lambda i, o, st: plan.exec_dev(i[0], nx, 0, acc0, delta, o[0], nout, st),
                       (plan,))
        if form == "batch":
            ldx = nx + 3
            return Run([(F32, ldx * ncols)], [(F32, nout * ncols)],
                       lambda i, o, st: plan.exec_batch_dev(i[0], nx, ldx, ncols, 0, acc0, delta, o[0], nout, st), (plan,))
        assert form == "stream"
        H = -(-ARB_HLEN // ARB_NPHASES) - 1
        return Run([(F32, H * ncols), (F32, nx * ncols)], [(F32, H * ncols), (F32, nout * ncols)],
                   lambda i, o, st: plan.stream_exec_dev(i[0], o[0], i[1], nx, ncols, 1, acc0, delta, o[1], nout, nout, st),
                   (plan,))
    return build


# ---- plan-less calls

def _conv_nd(form):
    def build(dsp, scale):
        if form == "os":
            us, vs, nffts = (200 * scale, 150), (9, 7), (32, 32)
        else:
            us, vs = (40 * scale, 30), (7, 5)
            nffts = None if form == "direct" else tuple(a + b - 1 for a, b in zip(us, vs))
        no = int(np.prod([a + b - 1 for a, b in zip(us, vs)]))
        return Run([(F32, int(np.prod(us))), (F32, int(np.prod(vs)))], [(F32, no)],
                   lambda i, o, st: dsp._lib.conv_nd_dev(F32, us, i[0], vs, i[1], nffts, o[0], form == "os", st))
    return build


def _hilbert(dsp, scale):
    n, ncols = 1000 * scale + 1, 3
    return Run([(F32, n * ncols)], [(C64, n * ncols)], lambda i, o, st: dsp._lib.hilbert_dev(F32, i[0], n, ncols, o[0], st))


def _per2(ptype):
    def build(dsp, scale):
        shape, nfft, r = (37 * scale, 50), (64 * scale, 64), 2.5 * 37 * scale * 50
        nout = nfft[0] * nfft[1] if ptype == 0 else min(nfft) // 2 + 1
        compare = None
        if ptype:                    # Float64 atomics add the rings in a run-to-run order: the kernel-path suite's bound
            def compare(got, ref, data):
                S, E = ck.per2_ref(data[0].reshape(shape, order="F"), nfft[0], nfft[1], F32)
                tot, bnd, pop, kmax = ck.radial_ref(S, E, nfft[0], nfft[1], r, F32)
                err = np.abs(got[0].astype(np.float64) - tot)
                return got[0].size == kmax and bool(np.all(err <= bnd))
        return Run([(F32, shape[0] * shape[1])], [(F32, nout)],
                   lambda i, o, st: dsp._lib.periodogram2_dev(F32, i[0], shape, nfft, r, ptype, o[0], st), compare=compare)
    return build


def _cases():
    c = [Case("fir", ["dspb200_fir_exec_dev"], "fir", _fir(False)),
         Case("fir-state", ["dspb200_fir_exec_state_dev"], "fir", _fir(True))]
    for dt, nv, nfft, form, entry in ((F32, 100, 0, "plain", "dspb200_os_exec_dev"),
                                      (C64, 37, 1000, "plain", "dspb200_os_exec_dev"),
                                      (F32, 100, 0, "range", "dspb200_os_exec_range_dev"),
                                      (F32, 100, 0, "state", "dspb200_os_exec_state_dev"),
                                      (F32, 9000, 0, "state", "dspb200_os_exec_state_dev")):
        route = _os_route(dt, nv, nfft)
        c.append(Case(f"os-{form}-{route}", [entry], ("os-state/" if form == "state" else "os/") + route,
                      _os(dt, nv, nfft, form)))
    spec_forms = (("welch", ["dspb200_welch_exec_dev"], "welch/single"),
                  ("batch", ["dspb200_welch_batch_exec_dev"], "welch/batched"),
                  ("range", ["dspb200_welch_exec_range_dev"], "welch/single"),
                  ("triple", ["dspb200_welch_begin_dev", "dspb200_welch_accumulate_dev", "dspb200_welch_finalize_dev"],
                   "welch/single"),
                  ("stft", ["dspb200_stft_exec_dev"], "stft"),
                  ("stft_stream", ["dspb200_stft_stream_exec_dev"], "stft"),
                  ("welch_stream", ["dspb200_welch_stream_exec_dev"], "welch/batched"),
                  ("welch_stream_power", ["dspb200_welch_stream_power_dev"], "finalize"))
    mt_forms = (("pgram", "dspb200_mt_pgram_exec_dev"), ("spectrogram", "dspb200_mt_spectrogram_exec_dev"),
                ("pgram_batch", "dspb200_mt_pgram_batch_exec_dev"),
                ("spectrogram_batch", "dspb200_mt_spectrogram_batch_exec_dev"), ("cross", "dspb200_mt_cross_spectra_exec_dev"))
    for dt, nfft in ((F32, 1024), (F32, 1000)):
        sr = _spec_route(dt, nfft)
        for form, entries, kernel in spec_forms:
            if form == "stft" and sr == "fused":
                kernel = "stft/" + _stft_route(dt, nfft)
            c.append(Case(f"{form}-{nfft}", entries, f"spectral/{sr} {kernel}" if sr == "fused" else f"spectral/{sr}",
                          _spec(dt, nfft, form)))
        for form, entry in mt_forms:
            c.append(Case(f"mt-{form}-{nfft}", [entry], f"spectral/{sr}", _mt(dt, nfft, form)))
    c.append(Case("stft-c64-2048", ["dspb200_stft_exec_dev"], "spectral/fused stft/" + _stft_route(C64, 2048),
                  _spec(C64, 2048, "stft")))
    for fam, (I, D, hlen) in RS_FAMILIES.items():
        c.append(Case(f"resample-{fam}", ["dspb200_resample_exec_dev"], "rs/" + rk.expected_family(I, D, hlen, F32, F32, 2),
                      _rs(I, D, hlen, "plain")))
    c += [Case("resample-range", ["dspb200_resample_exec_range_dev"], "rs/" + rk.expected_family(3, 2, 38, F32, F32),
               _rs(3, 2, 38, "range")),
          Case("resample-stream", ["dspb200_resample_stream_exec_dev"], "rs/" + rk.expected_family(3, 2, 38, F32, F32, 2),
               _rs(3, 2, 38, "stream")),
          Case("arb", ["dspb200_resample_arb_exec_dev"], "arb", _arb("plain")),
          Case("arb-batch", ["dspb200_resample_arb_batch_exec_dev"], "arb", _arb("batch")),
          Case("arb-stream", ["dspb200_resample_arb_stream_exec_dev"], "arb", _arb("stream")),
          Case("conv-nd-fft", ["dspb200_conv_nd_exec_dev"], "plan-less", _conv_nd("fft")),
          Case("conv-nd-direct", ["dspb200_conv_nd_exec_dev"], "plan-less", _conv_nd("direct")),
          Case("conv-nd-os", ["dspb200_conv_nd_os_exec_dev"], "plan-less", _conv_nd("os")),
          Case("hilbert", ["dspb200_hilbert_exec_dev"], "plan-less", _hilbert),
          Case("periodogram2-full", ["dspb200_periodogram2_exec_dev"], "plan-less", _per2(0)),
          Case("periodogram2-radial", ["dspb200_periodogram2_exec_dev"], "plan-less", _per2(1))]
    return c


CASES = _cases()
ASYNC_CASES = [c for c in CASES if not c.sync]
# one async case per family plus the plan-less calls: what every thread of the thread test runs
THREAD_CASES = [c for c in CASES if c.name in ("fir", "os-plain-fused", "welch-1024", "stft-1024", "resample-mp2",
                                               "arb-batch", "mt-pgram_batch-1024", "conv-nd-fft", "conv-nd-os", "hilbert",
                                               "periodogram2-full")]


def _ids(cases):
    return [c.name for c in cases]


# =============================================================================== CPU tests

def test_header_classifies_every_dev_entry_point():
    kinds = header_dev_entry_points()
    assert len(kinds) == 30, sorted(kinds)
    assert "dspb200_set_device" not in kinds
    assert {k for k, v in kinds.items() if v == "sync"} == SYNC_ENTRIES
    with open(HEADER) as f:
        text = f.read()
    # the conventions block says which _dev calls a CUDA graph may capture
    assert re.search(r"captured\s+in\s+a\s+CUDA\s+graph", text)


def test_case_table_covers_every_entry_point_and_route():
    kinds = header_dev_entry_points()
    covered = {e for c in CASES for e in c.entries}
    assert covered == set(kinds), (sorted(set(kinds) - covered), sorted(covered - set(kinds)))
    assert len({c.name for c in CASES}) == len(CASES)
    for c in CASES:                  # a case's entries share one class: the sync flag is that of all of them
        assert {kinds[e] for e in c.entries} == {"sync" if c.sync else "async"}, c.name
    routes = {c.route for c in CASES}
    want = {"os/fused", "os/generic", "os-state/fused", "os-state/generic", "rs/mp2", "rs/mp", "rs/tiled", "rs/generic",
            "spectral/cufft", "spectral/fused welch/single", "spectral/fused welch/batched", "spectral/fused stft/w1k",
            "spectral/fused stft/fused"}
    assert want <= routes, sorted(want - routes)
    for c in CASES:                  # every spectral entry point at a fused and a cuFFT size
        if c.route.startswith("spectral/fused"):
            twin = c.name.replace("1024", "1000")
            assert c.name == "stft-c64-2048" or any(d.name == twin and d.route == "spectral/cufft" for d in CASES), c.name
    assert {c.entries[0] for c in THREAD_CASES} >= {"dspb200_conv_nd_exec_dev", "dspb200_conv_nd_os_exec_dev",
                                                     "dspb200_hilbert_exec_dev", "dspb200_periodogram2_exec_dev"}


def test_last_error_is_per_thread():
    """A refusal in one thread leaves another thread's message alone (the refusals fail before any CUDA call)."""
    dsp = pytest.importorskip("dspb200")
    lib = dsp._lib.lib
    barrier = threading.Barrier(2, timeout=60)
    seen, errors = {}, []

    def refuse(code):
        h = C.c_void_p(None)
        taps = np.ones(4, dtype=np.float32)
        rc = lib.dspb200_resample_plan_create(C.byref(h), code, 0, dsp._lib.ptr(taps), 4, 2, 1)
        assert rc == dsp._lib.EINVALID
        return dsp._lib.last_error()

    def worker(name, code, first):
        try:
            if first:
                seen[name, 0] = refuse(code)
            barrier.wait()
            if not first:
                seen[name, 0] = refuse(code)
            barrier.wait()
            seen[name, 1] = dsp._lib.last_error()
        except BaseException as e:       # reported by the main thread
            errors.append(e)
            barrier.abort()

    main_before = dsp._lib.last_error()
    ts = [threading.Thread(target=worker, args=("a", 17, True)), threading.Thread(target=worker, args=("b", 19, False))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    assert "17" in seen["a", 0] and "19" in seen["b", 0]
    assert seen["a", 1] == seen["a", 0] and seen["b", 1] == seen["b", 0]
    assert dsp._lib.last_error() == main_before


# =============================================================================== GPU harness

@pytest.fixture(scope="module")
def dsp():
    return pytest.importorskip("dspb200")


class Pinned:
    """dspb200_host_alloc memory holding `n` elements of `dt`."""

    def __init__(self, dsp, dt, n):
        self.lib, self.dt, self.n = dsp._lib, np.dtype(dt), n
        self.nbytes = n * self.dt.itemsize
        p = C.c_void_p(None)
        self.lib.check(self.lib.lib.dspb200_host_alloc(C.byref(p), max(self.nbytes, 16)))
        self.ptr = p.value
        self.arr = np.frombuffer((C.c_char * max(self.nbytes, 16)).from_address(self.ptr), dtype=self.dt, count=n)

    def close(self):
        if self.ptr:
            self.arr = None
            self.lib.lib.dspb200_host_free(self.ptr)
            self.ptr = None


class Bufs:
    """Device buffers of one Run: inputs between sentinel guards, holding sentinels until load(); outputs between NaN
    guards, NaN until written.  Inputs are copied in from pinned memory and outputs back into pinned memory."""

    def __init__(self, dsp, run, data, rng):
        self.lib = dsp._lib
        self.gin = [Guarded(dt, n, rng) for dt, n in run.ins]
        self.gout = [Guarded(dt, n) for dt, n in run.outs]
        self.pin = [Pinned(dsp, dt, n) for dt, n in run.ins]
        self.pout = [Pinned(dsp, dt, n) for dt, n in run.outs]
        self.iptr = [g.ptr for g in self.gin]
        self.optr = [g.ptr for g in self.gout]
        self.set_data(data)

    def set_data(self, data):
        self.data = data
        for p, x in zip(self.pin, data):
            p.arr[:] = x

    def load(self, st):
        for g, p in zip(self.gin, self.pin):
            if p.nbytes:
                self.lib.check(self.lib.lib.dspb200_memcpy_h2d(g.ptr, p.ptr, p.nbytes, st))

    def reset(self, st):
        """Sentinels back into the inputs and NaN into the outputs, as before the first load: a call that does not wait
        for the next load reads the sentinels, not the data an earlier load left behind."""
        for g in self.gin:
            self.lib.check(self.lib.lib.dspb200_memcpy_h2d(g.ptr, self.lib.ptr(g.host[g.lo:g.lo + g.n]), g.n * g.dt.itemsize,
                                                           st))
        self.clear_outputs(st)

    def clear_outputs(self, st):
        for g, p in zip(self.gout, self.pout):
            p.arr[:] = np.nan
            if p.nbytes:
                self.lib.check(self.lib.lib.dspb200_memcpy_h2d(g.ptr, p.ptr, p.nbytes, st))
        self.lib.check(self.lib.lib.dspb200_stream_sync(st))

    def fetch(self, st):
        for g, p in zip(self.gout, self.pout):
            if p.nbytes:
                self.lib.check(self.lib.lib.dspb200_memcpy_d2h(p.ptr, g.ptr, p.nbytes, st))

    def results(self):
        """The fetched outputs, after checking every guard cell (call after the stream has drained)."""
        for g in self.gin + self.gout:
            g.data()
        return [p.arr.copy() for p in self.pout]

    def close(self):
        for p in self.pin + self.pout:
            p.close()


class Ctx:
    """torch streams and the delay that holds a stream back: torch.cuda._sleep, calibrated against CUDA events, or a long
    time-domain FIR from the library where _sleep is missing."""

    def __init__(self, dsp, torch):
        self.dsp, self.torch, self.lib = dsp, torch, dsp._lib
        s = torch.cuda.Stream()
        self._fir = None
        if not hasattr(torch.cuda, "_sleep"):
            self._fir = self._fir_producer()
        cyc = 20_000_000
        with torch.cuda.stream(s):
            self._produce(s, cyc)                         # first launch: module load
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            self._produce(s, cyc)
            b.record(s)
        b.synchronize()
        self.units_per_s = cyc / (a.elapsed_time(b) * 1e-3)

    def _fir_producer(self):
        rng = np.random.default_rng(3)
        plan = self.lib.FirPlan(_sig(rng, F32, 4096))
        n = 1 << 20
        x, y = Guarded(F32, n, data=_sig(rng, F32, n)), Guarded(F32, n)
        return plan, x, y, n

    def _produce(self, s, units):
        if self._fir is None:
            with self.torch.cuda.stream(s):
                self.torch.cuda._sleep(int(units))
            return
        plan, x, y, n = self._fir                         # units: samples of a 4096-tap FIR
        for _ in range(max(1, int(units) // n)):
            plan.exec_dev(x.ptr, n, 1, y.ptr, s.cuda_stream)

    def delay(self, s, seconds):
        self._produce(s, seconds * self.units_per_s)

    def stream(self):
        return self.torch.cuda.Stream()

    def sync(self, st):
        self.lib.check(self.lib.lib.dspb200_stream_sync(st))


@pytest.fixture(scope="module")
def ctx(dsp):
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("torch has no CUDA device")
    return Ctx(dsp, torch)


def _rng(case, k=0):
    return np.random.default_rng([sum(map(ord, case.name)), len(case.name), k])


def reference(ctx, run, data):
    """The call on stream 0 (serialised with every blocking stream), then a synchronisation of stream 0."""
    b = Bufs(ctx.dsp, run, data, np.random.default_rng(1))
    try:
        b.load(None)
        run.call(b.iptr, b.optr, None)
        b.fetch(None)
        ctx.sync(None)
        return b.results()
    finally:
        b.close()


def warm(ctx, run, bufs, s):
    """One whole call on s (input, call, output); returns its host time, which sizes the delay."""
    t0 = time.perf_counter()
    bufs.load(s.cuda_stream)
    run.call(bufs.iptr, bufs.optr, s.cuda_stream)
    bufs.fetch(s.cuda_stream)
    ctx.sync(s.cuda_stream)
    return time.perf_counter() - t0


_ON_S = object()


def check_window(ctx, case, run, bufs, s, ref, delay_s, warm_s, call_stream=_ON_S, plant_sync=False):
    """Input copy behind the delay on s, the call, the output copy on s; the ordering, the asynchrony (or completion) and
    the delay-to-issue ratio are asserted.  call_stream / plant_sync plant misuse for the harness self-checks."""
    ctx.delay(s, delay_s)
    bufs.load(s.cuda_stream)
    st = s.cuda_stream if call_stream is _ON_S else call_stream
    t0 = time.perf_counter()
    run.call(bufs.iptr, bufs.optr, st)
    issue = time.perf_counter() - t0
    if plant_sync:
        ctx.sync(s.cuda_stream)
    idle = s.query()
    if call_stream is not _ON_S:
        ctx.sync(call_stream)
    bufs.fetch(s.cuda_stream)
    ctx.sync(s.cuda_stream)
    got = bufs.results()
    assert run.same(got, ref, bufs.data), f"ordering: {case.name} does not equal the stream-0 call"
    if case.sync:
        assert delay_s >= ISSUE_RATIO * warm_s, (case.name, delay_s, warm_s)
        assert idle, f"completion: {case.name} returned before its work on the stream had completed"
    else:
        assert delay_s >= ISSUE_RATIO * issue, f"delay {delay_s:.4f} s is not {ISSUE_RATIO}x the issue time {issue:.5f} s"
        assert not idle, f"asynchrony: the stream was idle when {case.name} returned"
    return issue


def _delay_for(warm_s):
    return max(DELAY_OVER_WARM * warm_s, MIN_DELAY)


# =============================================================================== GPU tests

@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_ids(CASES))
def test_caller_stream_order_and_no_remembered_stream(dsp, ctx, case):
    """Ordering and asynchrony on S1, then the same plan on S2 and back on S1 (each after the previous stream drained)."""
    run = case.build(dsp, 1)
    data = run.inputs(_rng(case))
    ref = reference(ctx, run, data)
    s1, s2 = ctx.stream(), ctx.stream()
    bufs = Bufs(dsp, run, data, _rng(case, 1))
    try:
        warm_s = max(warm(ctx, run, bufs, s) for s in (s1, s2, s1))
        assert run.same(bufs.results(), ref, data), f"{case.name}: the warm call on a torch stream differs"
        delay_s = _delay_for(warm_s)
        for s in (s1, s2, s1):
            bufs.reset(None)
            check_window(ctx, case, run, bufs, s, ref, delay_s, warm_s)
    finally:
        bufs.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_ids(CASES))
def test_two_plans_at_once(dsp, ctx, case):
    """Plan A queued behind a delay on S1, a larger plan B of the same entry point issued and finished on S2 meanwhile."""
    ra, rb = case.build(dsp, 1), case.build(dsp, 2)
    da, db = ra.inputs(_rng(case, 2)), rb.inputs(_rng(case, 3))
    refa, refb = reference(ctx, ra, da), reference(ctx, rb, db)
    s1, s2 = ctx.stream(), ctx.stream()
    ba, bb = Bufs(dsp, ra, da, _rng(case, 4)), Bufs(dsp, rb, db, _rng(case, 5))
    try:
        warm_s = warm(ctx, ra, ba, s1) + warm(ctx, rb, bb, s2)
        delay_s = _delay_for(warm_s)
        ba.reset(None)
        bb.reset(None)
        ctx.delay(s1, delay_s)
        ba.load(s1.cuda_stream)
        ra.call(ba.iptr, ba.optr, s1.cuda_stream)
        bb.load(s2.cuda_stream)
        rb.call(bb.iptr, bb.optr, s2.cuda_stream)
        bb.fetch(s2.cuda_stream)
        ctx.sync(s2.cuda_stream)
        if not case.sync:
            assert not s1.query(), f"{case.name}: plan A finished before plan B although it waits behind the delay"
        ba.fetch(s1.cuda_stream)
        ctx.sync(s1.cuda_stream)
        assert rb.same(bb.results(), refb, db), f"{case.name}: plan B differs"
        assert ra.same(ba.results(), refa, da), f"{case.name}: plan A differs"
    finally:
        ba.close()
        bb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ASYNC_CASES, ids=_ids(ASYNC_CASES))
def test_cuda_graph_capture_and_replay(dsp, ctx, case):
    """Warm up with the captured shapes and pointers, capture on a side stream, write new input into the same buffers and
    replay twice: each replay equals an eager call on the new input."""
    torch = ctx.torch
    run = case.build(dsp, 1)
    d0, d1 = run.inputs(_rng(case, 6)), run.inputs(_rng(case, 7))
    ref1 = reference(ctx, run, d1)
    s = ctx.stream()
    bufs = Bufs(dsp, run, d0, _rng(case, 8))
    try:
        for _ in range(2):
            warm(ctx, run, bufs, s)
        g = torch.cuda.CUDAGraph()
        gc.collect()
        gc.disable()                 # a plan destroyed by the collector would free device memory inside the capture
        try:
            with torch.cuda.graph(g, stream=s):
                run.call(bufs.iptr, bufs.optr, torch.cuda.current_stream().cuda_stream)
        finally:
            gc.enable()
        bufs.set_data(d1)
        bufs.load(s.cuda_stream)
        ctx.sync(s.cuda_stream)
        for rep in range(2):
            bufs.clear_outputs(s.cuda_stream)
            with torch.cuda.stream(s):
                g.replay()
            bufs.fetch(s.cuda_stream)
            ctx.sync(s.cuda_stream)
            assert run.same(bufs.results(), ref1, d1), f"{case.name}: replay {rep} differs from the eager call"
        del g
    finally:
        bufs.close()


@pytest.mark.gpu
def test_four_threads_plans_and_plan_less_calls(dsp, ctx):
    """Four threads, each with its own plans and stream, run one async case per family and the plan-less calls (which
    share the cuFFT plan cache and the scratch arena) three times over; every output equals the serial reference."""
    nthreads, reps = 4, 3
    datas = [run_case.build(dsp, 1).inputs(_rng(run_case, 9)) for run_case in THREAD_CASES]
    refs = [reference(ctx, c.build(dsp, 1), d) for c, d in zip(THREAD_CASES, datas)]
    work = []
    for t in range(nthreads):
        runs = [c.build(dsp, 1) for c in THREAD_CASES]
        work.append((ctx.stream(), runs, [Bufs(dsp, r, d, _rng(c, 10 + t)) for r, d, c in zip(runs, datas, THREAD_CASES)]))
    barrier = threading.Barrier(nthreads, timeout=120)
    got, errors = {}, []

    def worker(t):
        s, runs, bufs = work[t]
        try:
            barrier.wait()
            for rep in range(reps):
                for k, (r, b) in enumerate(zip(runs, bufs)):
                    b.load(s.cuda_stream)
                    r.call(b.iptr, b.optr, s.cuda_stream)
                    b.fetch(s.cuda_stream)
                    ctx.sync(s.cuda_stream)
                    got[t, rep, k] = [p.arr.copy() for p in b.pout]
        except BaseException as e:
            errors.append(e)
            barrier.abort()

    ts = [threading.Thread(target=worker, args=(t,)) for t in range(nthreads)]
    try:
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert not errors, errors
        for (t, rep, k), out in sorted(got.items()):
            c = THREAD_CASES[k]
            assert work[t][1][k].same(out, refs[k], datas[k]), (c.name, t, rep)
        assert len(got) == nthreads * reps * len(THREAD_CASES)
        for _, _, bufs in work:
            for b in bufs:
                b.results()
    finally:
        for _, _, bufs in work:
            for b in bufs:
                b.close()


def _host_calls(dsp, rng):
    """Host-pointer calls of distinct plans: [(name, fn() -> list of outputs)], inputs fixed by rng."""
    L = dsp._lib
    taps = _sig(np.random.default_rng(5), F32, 65)
    x = _sig(rng, F32, (1 << 22) + 4097)
    nx2, ncols = 300_001, 3
    x2 = np.asfortranarray(_sig(rng, F32, nx2 * ncols).reshape(nx2, ncols, order="F"))
    fir, os_, rs = L.FirPlan(taps), L.OsPlan(taps, 0), L.ResamplePlan(F32, taps, 3, 2)
    spec = L.SpecPlan(F32, 1024, 512, 1024, True, kp.window_of("hann", 1024, None))
    fw_os, fw_spec = L.OsPlan(taps, 0), L.SpecPlan(F32, 1024, 512, 1024, True, kp.window_of("hann", 1024, None))
    px = Pinned(dsp, F32, x.size)
    px.arr[:] = x
    k = spec.nsegments(x.size)

    def fir_call():
        out = np.empty_like(x2)
        fir.exec(x2, out)
        return [out]

    def os_call():
        out = np.empty((nx2 + 64, ncols), dtype=np.float32, order="F")
        os_.exec(x2, out, nx2, ncols, nx2 + 64)
        return [out]

    def rs_call():
        nout = nx2 * 3 // 2
        out = np.empty((nout, ncols), dtype=np.float32, order="F")
        rs.exec(x2, nx2, ncols, 4, 0, out, nout)
        return [out]

    def welch_call():
        out = np.empty(spec.nout, dtype=np.float32)
        spec.welch(x, 3.0 * k, out)
        return [out]

    def filt_welch_call():
        out = np.empty(fw_spec.nout, dtype=np.float32)
        fw_spec.filt_welch_ptr(fw_os, px.ptr, x.size, 3.0 * k, L.ptr(out))
        return [out]

    calls = [("fir", fir_call), ("os", os_call), ("resample", rs_call), ("welch", welch_call), ("filt_welch", filt_welch_call)]
    return calls, (fir, os_, rs, spec, fw_os, fw_spec), px


@pytest.mark.gpu
def test_host_pointer_calls_from_two_threads(dsp, ctx):
    """Host-pointer calls with distinct plans (each with its own staging pipe) from two threads at once equal the serial
    results."""
    data_seed = 11
    ref_calls, keep, ref_px = _host_calls(dsp, np.random.default_rng(data_seed))
    try:
        refs = {name: fn() for name, fn in ref_calls}
    finally:
        ref_px.close()
    sets = [_host_calls(dsp, np.random.default_rng(data_seed)) for _ in range(2)]
    barrier = threading.Barrier(2, timeout=120)
    got, errors = {}, []

    def worker(t):
        calls = sets[t][0]
        try:
            barrier.wait()
            for rep in range(2):
                for name, fn in (calls if t == 0 else calls[::-1]):
                    got[t, rep, name] = fn()
        except BaseException as e:
            errors.append(e)
            barrier.abort()

    ts = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    try:
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert not errors, errors
        assert len(got) == 2 * 2 * len(refs)
        for (t, rep, name), out in got.items():
            assert all(same_bits(a, b) for a, b in zip(out, refs[name])), (name, t, rep)
    finally:
        for _, _, px in sets:
            px.close()


# ---- the harness's own checks fail on planted misuse

def _planted(dsp, ctx, name):
    case = next(c for c in CASES if c.name == name)
    run = case.build(dsp, 1)
    data = run.inputs(_rng(case))
    ref = reference(ctx, run, data)
    s = ctx.stream()
    bufs = Bufs(dsp, run, data, _rng(case, 1))
    warm_s = warm(ctx, run, bufs, s)
    bufs.reset(None)
    return case, run, bufs, s, ref, _delay_for(warm_s), warm_s


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fir", "welch-1024", "resample-mp2"])
def test_planted_call_on_stream_zero_fails_the_ordering_check(dsp, ctx, name):
    """The call on stream 0 while its input arrives on S does not wait for the copy: it reads the sentinels."""
    case, run, bufs, s, ref, delay_s, warm_s = _planted(dsp, ctx, name)
    try:
        with pytest.raises(AssertionError, match="ordering"):
            check_window(ctx, case, run, bufs, s, ref, delay_s, warm_s, call_stream=None)
    finally:
        bufs.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fir", "welch-1024", "resample-mp2"])
def test_planted_stream_sync_fails_the_asynchrony_check(dsp, ctx, name):
    """A dspb200_stream_sync(S) inside the call window: the result is right, the asynchrony check fails."""
    case, run, bufs, s, ref, delay_s, warm_s = _planted(dsp, ctx, name)
    try:
        with pytest.raises(AssertionError, match="asynchrony"):
            check_window(ctx, case, run, bufs, s, ref, delay_s, warm_s, plant_sync=True)
    finally:
        bufs.close()
