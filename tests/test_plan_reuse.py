"""Every plan across sequences of differing calls: each call bit-identical to a fresh plan and exact on integer data.

Callers create a plan once and reuse it for many calls, and the front ends cache plans for them (`_OS_PLANS`, a
WelchConfig's SpecPlan, FIRFilter's plan per eltype, the plan-less calls' cuFFT plan cache and scratch arena).  Plans keep
state from one call to the next: launch configurations cached per alignment class (`welch_cfg`, `welch_batch_cfg`,
`welch_mt_cfg`, `fused_per_sm`, `arb_attr_set`), the rows of an open Welch accumulation (`rows_used`, `partial`, with
`fresh_from` deciding which rows a launch overwrites) and grow-only scratch (`bpartial`, `tmp`, `seam`, the host pipes, the
arena).  The kernel-path suites build a fresh plan per case or repeat one call; a stale configuration, a partial row left
by an earlier accumulation or a buffer sized by an earlier call would give wrong numbers there unnoticed.

Each sequence below runs on one plan.  After every call the same call -- same arguments, same device buffers, so the same
alignment -- runs on a freshly created plan with the same parameters (and the same pins), and the two results must agree
bit for bit; the kernel-path suites validate the fresh plan's result.  A Welch finalize depends on its whole
begin ... finalize sequence, so its fresh plan runs the same accumulate calls and nothing in between.  Integer data must
besides give the exact integer result (np.convolve, the direct polyphase sum), and spectral results must stay within the
per-bin bound of test_spectral_kernel_paths.py -- which catches what a defect shared by both plans would hide.  The radial
2-D periodogram adds Float64 atomics in a run-to-run order and is checked against its bound instead of for identity.
The plan-less calls have no plan: a revisited call must equal its first run.  Device inputs sit between sentinel cells
and must come back unchanged; outputs sit between NaN cells.  One refused call per plan kind (EINVALID before any launch)
must leave the plan as it was.

The CPU part builds the seeded sequences, restates the state each call touches (alignment class, whether Welch rows are
overwritten or added to, the bytes each grow-only buffer needs, the cuFFT plan-cache keys and their LRU order) and shows
that the sequences reach every transition listed in TRANSITIONS."""
import math
from fractions import Fraction

import numpy as np
import pytest

import test_client_kernel_paths as ck
import test_os_kernel_paths as osk
import test_resample_kernel_paths as rk
import test_spectral_kernel_paths as kp
from test_spectral_kernel_paths import F32, F64, C64, same_bits

GUARD_ALIGN = 16
PLAN_CACHE = 32                     # plans the plan-less calls' cuFFT cache keeps (runtime.cu, plan_cache_get)
ARENA_KEEP = 256 << 20              # arena buffers larger than this are released after each plan-less call (scratch_trim)
INDEX_LIMIT = 1 << 61               # DSPB200_INDEX_LIMIT
DEFAULT_BUDGET = ck.DEFAULT_BUDGET  # g_nd_os_budget


def cdiv(a, b):
    return -(-a // b)


# =============================================================================== sequences (CPU: plain data)
#
# A sequence is a list of ops, dicts with an "op" name and the call's sizes.  Buffers are placed at `off` elements past a
# 256-byte aligned address, which fixes every call's alignment class.

# ---- 1. overlap-save plans: (dtype, nfft, nv)
OS_INSTANCES = [(F32, 1024, 129), (F32, 16384, 4097), (C64, 16384, 4097), (F64, 8192, 1025), (F32, 3000, 501)]


def _os_id(inst):
    dt, N, nv = inst
    return f"{dt.name}-{N}-nv{nv}"


def os_sequence(inst):
    dt, N, nv = inst
    L = N - nv + 1
    co = osk.chunk_out(dt.itemsize, L)
    long_nu = 2 * co + L // 2 + 7
    first = dict(op="dev", ncols=70, nu=L + 3, nout=L + 3 + nv - 1, off=0)
    return [first,
            dict(op="dev", ncols=1, nu=5 * L + 7, nout=5 * L + 7, off=1),
            dict(op="range", u_begin=2 * L + 1, nu=3 * L + 1, out_begin=L // 2 + 5, count=2 * L + 9, off=0),
            dict(op="state", ncols=3, nx=2 * L + 11, si=True),
            dict(op="state", ncols=2, nx=L + 1, si=False),
            dict(op="host", ncols=1, nu=long_nu, nout=long_nu + nv - 1),
            dict(op="host", ncols=2, nu=L // 3 + 2, nout=L // 3 + 2 + nv - 1),
            dict(op="refuse", what="state si_in == si_out"),
            dict(op="dev", ncols=1, nu=5 * L + 7, nout=5 * L + 7, off=1),
            dict(first)]


def os_touch(inst, op):
    """What one overlap-save call touches: the occupancy cache of the fused kernel (stateless or stateful instance), and
    for host calls the bytes one slot of the host pipe stages (one chunk of about 32 MiB of outputs when the call is
    chunked, the whole call otherwise)."""
    dt, N, nv = inst
    L = N - nv + 1
    esz = dt.itemsize
    t = dict(form=op["op"], fused=osk.os_fused_ok(N, nv, dt == F64))
    if op["op"] == "host":
        chunked = osk.host_chunked(op["ncols"], op["nu"], op["nout"], esz, L)
        t["chunked"] = chunked
        nout = osk.chunk_out(esz, L) if chunked else op["nout"] * op["ncols"]
        t["pipe_bytes"] = (nout + nv - 1) * esz + nout * esz if chunked else (op["nu"] * op["ncols"] + nout) * esz
    if op["op"] in ("dev", "range", "state"):
        t["occupancy"] = "state" if op["op"] == "state" else "plain"
    return t


# front-end cache: fftfilt / conv through _OS_PLANS (8 plans, the oldest evicted first)
FRONT_TAPS = 9


def front_sequence():
    ops = [dict(op="fftfilt_host", taps=0, nx=50_001, ncols=2),
           dict(op="conv_dev", taps=0, nu=40_003),
           dict(op="fftfilt_dev", taps=0, nx=30_011, ncols=3),
           dict(op="conv_host", taps=0, nu=20_007)]
    ops += [dict(op="fftfilt_host", taps=t, nx=10_007 + t, ncols=1) for t in range(1, FRONT_TAPS)]
    ops += [dict(op="fftfilt_host", taps=0, nx=50_001, ncols=2), dict(op="conv_dev", taps=0, nu=40_003)]
    return ops


def front_cache_model(ops, cap=8):
    """_OS_PLANS restated: insertion order, the oldest popped when a ninth key arrives.  Per op: (hit, evicted key)."""
    cache, out = [], []
    for op in ops:
        k = op["taps"]
        if k in cache:
            out.append((True, None))
            continue
        ev = cache.pop(0) if len(cache) >= cap else None
        cache.append(k)
        out.append((False, ev))
    return out


# ---- 2. Welch on a spec plan: (dtype, nfft = n, hop)
WELCH_PLANS = [(F32, 4096, 2048), (F32, 1000, 500)]
WELCH_BATCH_SCRATCH = 32 << 20


def _wid(p):
    return f"{p[0].name}-{p[1]}"


def welch_batch_rows_cap(dt, N):
    return WELCH_BATCH_SCRATCH // (N * dt.itemsize)


def welch_sequence(wp):
    dt, N, hop = wp
    fused = kp.fused_size_ok(N, False)
    k = 37
    nchan = welch_batch_rows_cap(dt, N) + 52 if fused else 7       # fused: past the 32 MiB of partial rows, two groups
    ops = [dict(op="welch", k=k, off=0), dict(op="welch", k=k + 4, off=1), dict(op="welch", k=k, off=0),
           dict(op="welch", k=k - 6, off=1),
           dict(op="acc", k=60, chunks=[(0, 7, 0), (7, 15, 1)], batch=dict(nchan=nchan, k=1, off=0),
                rest=[(15, 33, 0), (33, 60, 1)]),
           dict(op="acc", k=23, chunks=[(0, 23, 1)], batch=None, rest=[]),
           dict(op="filt_welch", k=41), dict(op="host_welch", k=kp.host_chunk_segs(dt.itemsize, hop, 1 << 30) + 9),
           dict(op="filt_welch", k=19), dict(op="host_welch", k=11)]
    if fused:
        ops += [dict(op="pin", batched=0, mode=1, groups=1, vctas=24), dict(op="welch", k=k, off=0),
                dict(op="welch", k=k, off=1),
                dict(op="pin", batched=1, mode=0, groups=1, vctas=6), dict(op="batch", nchan=5, k=9, off=0),
                dict(op="acc", k=30, chunks=[(0, 9, 0)], batch=dict(nchan=3, k=4, off=1), rest=[(9, 30, 0)]),
                dict(op="pin", batched=0, mode=-1, groups=0, vctas=0), dict(op="welch", k=k, off=0),
                dict(op="pin", batched=1, mode=-1, groups=0, vctas=0)]
    ops += [dict(op="refuse", what="accumulate past the index domain", k=40, chunks=[(0, 11, 0)], rest=[(11, 40, 1)]),
            dict(op="batch", nchan=4, k=6, off=1), dict(op="welch", k=k, off=0)]
    return ops


def welch_class(dt, hop, n, off, seg0=0, sample_offset=0):
    """Alignment class of a single-signal Welch launch (launch_welch_fused): the first segment's start, hop and n."""
    esz = dt.itemsize
    return int(((off + seg0 * hop - sample_offset) * esz) % 16 == 0 and (hop * esz) % 16 == 0 and (n * esz) % 16 == 0)


def welch_batch_class(dt, hop, n, off, length, nchan):
    """welch_batch_aligned: base, channel stride (unless one channel), hop and n."""
    esz = dt.itemsize
    return int((off * esz) % 16 == 0 and ((length * esz) % 16 == 0 or nchan == 1) and (hop * esz) % 16 == 0
               and (n * esz) % 16 == 0)


def welch_touch(wp, op):
    """The Welch state one op touches: per launch, the (form, alignment class) whose configuration it uses and whether it
    writes (first launch after welch_begin) or adds to the partial rows; for a batch, the bytes of `bpartial` it needs and
    the channel groups it runs in (fused sizes)."""
    dt, N, hop = wp
    n, fused = N, kp.fused_size_ok(N, False)
    t = dict(launches=[], batch=None)
    name = op["op"]
    if name == "welch":
        t["launches"].append(("single", welch_class(dt, hop, n, op["off"]), "write"))
    if name in ("acc", "refuse"):
        first = True
        for b, e, off in op["chunks"]:
            t["launches"].append(("single", welch_class(dt, hop, n, off, b, b * hop), "write" if first else "add"))
            first = False
        if op.get("batch"):
            t["batch"] = _batch_touch(dt, N, hop, op["batch"], fused)
        for b, e, off in op["rest"]:
            t["launches"].append(("single", welch_class(dt, hop, n, off, b, b * hop), "add"))
    if name == "batch":
        t["batch"] = _batch_touch(dt, N, hop, op, fused)
    return t


def _batch_touch(dt, N, hop, b, fused):
    length = (b["k"] - 1) * hop + N
    cap = welch_batch_rows_cap(dt, N)
    groups = cdiv(b["nchan"], min(b["nchan"], cap)) if fused else b["nchan"]
    return dict(cls=welch_batch_class(dt, hop, N, b["off"], length, b["nchan"]), groups=groups,
                bpartial=min(b["nchan"], cap) * N * dt.itemsize if fused else 0)


# ---- 3. STFT: (dtype, nfft = n, hop)
STFT_PLANS = [(F32, 1024, 256), (C64, 2048, 512)]


def stft_sequence(sp):
    dt, N, hop = sp
    return [dict(op="stft", psd=0, k=9, nchan=3), dict(op="stream", nhist=0, nseg=6, extra=5, nchan=3, psd=0),
            dict(op="stft", psd=1, k=7, nchan=2), dict(op="stream", nhist=N - hop, nseg=9, extra=3, nchan=3, psd=1),
            dict(op="stft_acc", k=5, nchan=3), dict(op="stream", nhist=N - hop, nseg=4, extra=hop - 1, nchan=1, psd=0),
            dict(op="refuse", what="hist_out overlaps x"), dict(op="stft", psd=0, k=9, nchan=3)]


def stft_touch(sp, op):
    """One-shot calls are streams over an empty history; a stream with a history reads the seam of its own call."""
    dt, N, hop = sp
    kind = "oneshot" if op["op"] in ("stft", "stft_acc") else op["op"]
    w1k = dt == F32 and N == 1024
    return dict(kind=kind, w1k=w1k, psd={"stft_acc": 3}.get(op["op"], op.get("psd")),
                seam=op["op"] == "stream" and op["nhist"] > 0)


# ---- 4. multitaper: (dtype, nfft = n, hop, ntapers)
MT_PLANS = [(F32, 1024, 512, 3), (F32, 1000, 500, 3)]


def mt_sequence(mp):
    return [dict(op="pgram", nchan=70), dict(op="pgram", nchan=1), dict(op="spec", nchan=5, k=6),
            dict(op="plain_batch", nchan=40, k=5), dict(op="spec", nchan=1, k=3), dict(op="pgram", nchan=3),
            dict(op="refuse", what="mt_pgram len != n"), dict(op="spec", nchan=2, k=4), dict(op="pgram", nchan=1)]


def mt_touch(mp, op):
    """Bytes of the grow-only buffers: `bpartial` (fused mt_pgram: one nfft row per (channel, taper slice)) and `tmp`
    (cuFFT mt_spectrogram: one taper's PSD matrices)."""
    dt, N, hop, nt = mp
    fused = kp.fused_size_ok(N, False)
    nout = N // 2 + 1
    t = dict(op=op["op"])
    if op["op"] == "pgram" and fused:
        t["bpartial"] = op["nchan"] * N * dt.itemsize
    if op["op"] == "spec" and not fused:
        t["tmp"] = op["nchan"] * op["k"] * nout * dt.itemsize
    return t


# ---- 5. resampling
RS_INSTANCES = [(3, 2, 38), (5, 7, 60)]


def rs_sequence(inst):
    return [dict(op="dev", ncols=4, nx=7001), dict(op="dev", ncols=1, nx=20011),
            dict(op="range", x_begin=500, nloc=6001, j_begin=300, count=8000),
            dict(op="stream", ncols=3, nx=4001, hist=True), dict(op="stream", ncols=2, nx=1500, hist=False),
            dict(op="host", ncols=2, nx=9001), dict(op="refuse", what="range past the index domain"),
            dict(op="dev", ncols=4, nx=7001)]


ARB = (32, 12 * 32, 1.37)            # nphases, hlen, rate


def arb_sequence():
    return [dict(op="stream", ncols=3, nx=6009), dict(op="batch", ncols=3, nx=5003), dict(op="stream", ncols=2, nx=1501),
            dict(op="plain", nx=4007), dict(op="refuse", what="stream ldo < nout", nx=3001), dict(op="batch", ncols=5, nx=2001),
            dict(op="stream", ncols=3, nx=6009)]


def arb_touch(op):
    """resample_arb_batch_kernel<.., HIST> opts in to its shared memory once per HIST (arb_attr_set) and the occupancy
    cache is keyed on HIST: streams run HIST = true, the batch and plain forms false."""
    return dict(hist=op["op"] == "stream") if op["op"] != "refuse" else {}


# ---- 6. FIR plans: (dtype, nb)
FIR_INSTANCES = [(F32, 33), (F64, 129)]


def fir_sequence(inst):
    return [dict(op="dev", ncols=70, nx=5007), dict(op="dev", ncols=1, nx=40_001), dict(op="dev", ncols=3, nx=9001),
            dict(op="state_dev", ncols=70, nx=3001, si=True), dict(op="state_dev", ncols=1, nx=20_003, si=False),
            dict(op="host", ncols=3, nx=30_007), dict(op="host_state", ncols=1, nx=12_001, si=True),
            dict(op="host", ncols=70, nx=1001), dict(op="dev", ncols=1, nx=40_001), dict(op="refuse", what="x overlaps out"),
            dict(op="dev", ncols=3, nx=9001)]


def fir_touch(inst, op):
    """Host calls stage x, out and the state through the plan's buffers (grow-only) on the stream made by the first host
    call; device calls use neither."""
    dt, nb = inst
    esz = dt.itemsize
    if op["op"] in ("host", "host_state"):
        return dict(host=True, bytes=op["nx"] * op["ncols"] * esz)
    return dict(host=False)


# ---- 7. plan-less calls
def fft_type(real_in, f64, forward):
    """The cufftType of a transform (fft_type, cufft_exec.cuh), by name."""
    if real_in:
        return ("D2Z" if f64 else "R2C") if forward else ("Z2D" if f64 else "C2R")
    return "Z2Z" if f64 else "C2C"


def planless_keys(op):
    """The cuFFT plan-cache keys one plan-less call asks for, in order (plan_cache_get: rank, dims slowest first, embed,
    idist, odist, type, batch)."""
    kind = op["op"]
    if kind == "conv_fft":
        nf = tuple(reversed(op["nffts"]))
        return [(len(nf), nf, False, 0, 0, "R2C", 1), (len(nf), nf, False, 0, 0, "C2R", 1)]
    if kind == "conv_os":
        nf = tuple(reversed(op["nffts"]))
        keys = [(len(nf), nf, False, 0, 0, "R2C", 1)]
        b = conv_os_batch(op, op.get("budget", DEFAULT_BUDGET))
        if b > 1:
            keys.append((len(nf), nf, False, 0, 0, "R2C", b))
        keys.append((len(nf), nf, False, 0, 0, "C2R", b))
        return keys
    if kind == "hilbert":
        n = op["n"]
        return [(1, (n,), True, n, n, "R2C", op["ncols"]), (1, (n,), False, 0, 0, "C2C", op["ncols"])]
    assert kind == "per2"
    return [(2, (op["nfft"][1], op["nfft"][0]), False, 0, 0, "R2C", 1)]


def conv_os_batch(op, budget):
    """Blocks per batch of the N-D overlap-save path (conv_nd_dev, ND_OS), Float32."""
    nf, so = op["nffts"], [a + b - 1 for a, b in zip(op["us"], op["vs"])]
    nblocks = 1
    for f, v, o in zip(nf, op["vs"], so):
        nblocks *= cdiv(o, min(f - v + 1, o))
    nfe = int(np.prod(nf))
    nb = (nf[0] // 2 + 1) * int(np.prod(nf[1:]))
    per_block = nfe * 4 + nb * 8
    return max(1, min(budget // per_block, nblocks))


def conv_fft_arena(op):
    """Bytes of the arena slots 3 (real blocks), 4 and 5 (spectra) a Float32 conv_nd FFT call reserves."""
    nf = op["nffts"]
    nfe = int(np.prod(nf))
    nb = (nf[0] // 2 + 1) * int(np.prod(nf[1:]))
    return {3: nfe * 4, 4: nb * 8, 5: nb * 8}


def planless_cycle():
    """Plan-less calls with pairwise distinct cuFFT keys, enough of them that the first ones leave the cache."""
    ops = []
    for i, (a, b) in enumerate(((500, 41), (900, 132), (333, 17), (1201, 60), (77, 5), (2000, 99), (1500, 33), (257, 256),
                                   (4000, 7))):
        ops.append(dict(op="conv_fft", us=(a,), vs=(b,), nffts=(a + b - 1,), id=f"conv-fft-{a}"))
    for us, vs, nf in (((60, 40), (7, 5), (66, 44)), ((37, 23), (4, 9), (40, 31))):
        ops.append(dict(op="conv_fft", us=us, vs=vs, nffts=nf, id=f"conv-fft-{us[0]}x{us[1]}"))
    for us, vs, nf in (((200, 150), (9, 7), (32, 32)), ((300, 90), (13, 5), (64, 16))):
        ops.append(dict(op="conv_os", us=us, vs=vs, nffts=nf, id=f"conv-os-{us[0]}x{us[1]}"))
    for n, c in ((1000, 3), (1031, 2), (4096, 1), (65537, 1), (17, 64)):
        ops.append(dict(op="hilbert", n=n, ncols=c, id=f"hilbert-{n}x{c}"))
    for shape, nfft, pt in (((37, 50), (64, 64), 0), ((37, 50), (64, 64), 1), ((100, 30), (128, 40), 2),
                            ((20, 20), (30, 50), 0), ((64, 9), (64, 16), 1)):
        ops.append(dict(op="per2", shape=shape, nfft=nfft, ptype=pt, id=f"per2-{nfft[0]}x{nfft[1]}-{pt}"))
    return ops


def planless_sequence():
    cyc = planless_cycle()
    revisit = [dict(o) for o in cyc[:4]] + [dict(cyc[13]), dict(cyc[16])]
    arena = [dict(op="conv_fft", us=(3000, 3000), vs=(5, 5), nffts=(4096, 4096), id="arena-large", big=True),
             dict(op="conv_fft", us=(60, 40), vs=(7, 5), nffts=(66, 44), id="conv-fft-60x40"),
             dict(op="conv_fft", us=(500,), vs=(41,), nffts=(540,), id="conv-fft-500"),
             dict(op="conv_fft", us=(6000, 5000), vs=(3, 3), nffts=(8192, 9000), id="arena-trimmed", big=True),
             dict(op="conv_fft", us=(37, 23), vs=(4, 9), nffts=(40, 31), id="conv-fft-37x23"),
             dict(op="conv_fft", us=(3000, 3000), vs=(5, 5), nffts=(4096, 4096), id="arena-large", big=True)]
    os_op = dict(op="conv_os", us=(300, 90), vs=(13, 5), nffts=(64, 16))
    small = 2 * (64 * 16 * 4 + 33 * 16 * 8)
    budget = [dict(os_op, budget=DEFAULT_BUDGET, id="os-budget-default"),
              dict(os_op, op="set_budget", budget=small),
              dict(os_op, budget=small, id="os-budget-small"),
              dict(os_op, op="set_budget", budget=DEFAULT_BUDGET),
              dict(os_op, budget=DEFAULT_BUDGET, id="os-budget-default"),
              dict(op="refuse", what="nffts below size(v)")]
    return cyc + revisit + arena + budget


def lru_model(ops, cap=PLAN_CACHE):
    """The plan cache restated from empty: per op, the keys it finds (hits) and the keys its misses evict."""
    cache, clock, out = {}, 0, []
    for op in ops:
        if op["op"] not in ("conv_fft", "conv_os", "hilbert", "per2") or op.get("big"):
            out.append(dict(hits=[], evicted=[]))
            if op.get("big"):                   # the large calls ask for keys too (rank-2, batch 1)
                for k in planless_keys(op):
                    clock += 1
                    if k not in cache and len(cache) >= cap:
                        cache.pop(min(cache, key=cache.get))
                    cache[k] = clock
            continue
        hits, ev = [], []
        for k in planless_keys(op):
            clock += 1
            if k in cache:
                hits.append(k)
            elif len(cache) >= cap:
                old = min(cache, key=cache.get)
                cache.pop(old)
                ev.append(old)
            cache[k] = clock
        out.append(dict(hits=hits, evicted=ev))
    return out


# =============================================================================== transitions (CPU model)

def _grow_shrink(tag, sizes, out):
    """Tags for a grow-only buffer given the bytes each call needs: grown, reused by a smaller call, regrown."""
    cap = 0
    for i, s in enumerate(sizes):
        if s is None:
            continue
        if s > cap:
            out.add(f"{tag}:regrow" if cap and any(x is not None and x < cap for x in sizes[:i]) else f"{tag}:grow")
            cap = s
        elif s < cap:
            out.add(f"{tag}:reuse-smaller")


def reached_transitions():
    r = set()
    for inst in OS_INSTANCES:
        seq, tag = os_sequence(inst), f"os/{_os_id(inst)}"
        forms = [(o["op"], o.get("ncols"), o.get("si")) for o in seq]
        for a, b in zip(forms, forms[1:]):
            if a[0] == b[0] == "dev" and a[1] == 70 and b[1] == 1:
                r.add(f"{tag}:dev70->dev1")
        touches = [os_touch(inst, o) for o in seq]
        for o, t in zip(seq, touches):
            if o["op"] == "range":
                r.add(f"{tag}:range")
            if o["op"] == "state":
                r.add(f"{tag}:state+si" if o["si"] else f"{tag}:state-si")
            if o["op"] == "refuse":
                r.add("refuse:os")
        hosts = [t for t in touches if t["form"] == "host"]
        if len(hosts) >= 2 and hosts[0]["chunked"] and not hosts[1]["chunked"]:
            r.add(f"{tag}:host-chunked->host-short")
        _grow_shrink(f"{tag}:pipe", [t.get("pipe_bytes") for t in touches], r)
        occ = [t.get("occupancy") for t in touches if t.get("occupancy")]
        if "plain" in occ and "state" in occ and occ.index("state") < len(occ) - 1 - occ[::-1].index("plain"):
            r.add(f"{tag}:stateful->stateless")
    fs = front_sequence()
    model = front_cache_model(fs)
    if any(ev == 0 for _, ev in model):
        r.add("os-cache:evict")
        i = next(i for i, (_, ev) in enumerate(model) if ev == 0)
        if any(o["taps"] == 0 for o in fs[i + 1:]):
            r.add("os-cache:revisit-evicted")
    kinds = [o["op"] for o in fs[:4]]
    if {"fftfilt_host", "conv_dev", "fftfilt_dev", "conv_host"} <= set(kinds) and all(h for h, _ in model[1:4]):
        r.add("os-cache:host-dev-shared")
    for wp in WELCH_PLANS:
        tag = f"welch/{_wid(wp)}"
        seq = welch_sequence(wp)
        ts = [welch_touch(wp, o) for o in seq]
        cls = [t["launches"][0][1] for o, t in zip(seq, ts) if o["op"] == "welch"]
        if any(a != b for a, b in zip(cls, cls[1:])):
            r.add(f"{tag}:welch-class-alternates")
        for o, t in zip(seq, ts):
            if o["op"] == "acc" and o["batch"] and o["rest"]:
                if any(m == "write" for _, _, m in t["launches"]) and t["launches"][-1][2] == "add":
                    r.add(f"{tag}:acc->batch->acc")
                if t["batch"]["groups"] > 1 and kp.fused_size_ok(wp[1], False):
                    r.add(f"{tag}:batch-in-channel-groups")
            if o["op"] == "refuse":
                r.add("refuse:spec")
        _grow_shrink(f"{tag}:bpartial", [t["batch"]["bpartial"] if t["batch"] and t["batch"]["bpartial"] else None
                                          for t in ts], r)
        for name in ("filt_welch", "host_welch"):
            ks = [o["k"] for o in seq if o["op"] == name]
            if len(set(ks)) > 1:
                r.add(f"{tag}:{name}-lengths")
        for a, b in zip(seq, seq[1:]):
            if a["op"] == "pin" and b["op"] in ("welch", "batch"):
                r.add(f"{tag}:{'unpin' if a['mode'] < 0 else 'pin'}->call")
    for sp in STFT_PLANS:
        tag = f"stft/{_wid(sp)}"
        seq = stft_sequence(sp)
        ts = [stft_touch(sp, o) for o in seq]
        for a, b in zip(ts, ts[1:]):
            if a["kind"] != b["kind"] and "refuse" not in (a["kind"], b["kind"]):
                r.add(f"{tag}:{a['kind']}->{b['kind']}")
        psds = [t["psd"] for t in ts if t["kind"] == "oneshot"]
        if {0, 1, 3} <= set(psds):
            r.add(f"{tag}:raw-psd-acc")
        if any(t["seam"] for t in ts):
            r.add(f"{tag}:seam")
        if any(t["w1k"] for t in ts):
            r.add("stft:w1k")
        if any(o["op"] == "refuse" for o in seq):
            r.add("refuse:stft")
    for mp in MT_PLANS:
        tag = f"mt/{_wid(mp)}"
        seq = mt_sequence(mp)
        ts = [mt_touch(mp, o) for o in seq]
        _grow_shrink(f"{tag}:bpartial", [t.get("bpartial") for t in ts], r)
        _grow_shrink(f"{tag}:tmp", [t.get("tmp") for t in ts], r)
        ops = [(o["op"], o.get("nchan")) for o in seq]
        if ("pgram", 70) in ops and ("pgram", 1) in ops:
            r.add(f"{tag}:pgram-batch->vector")
        if ops.index(("spec", 5)) < ops.index(("spec", 1)):
            r.add(f"{tag}:spec-batch->vector")
        i = [o[0] for o in ops].index("plain_batch")
        if "pgram" in [o[0] for o in ops[:i]] and "pgram" in [o[0] for o in ops[i + 1:]]:
            r.add(f"{tag}:plain-batch-between")
        if any(o["op"] == "refuse" for o in seq):
            r.add("refuse:mt")
    for inst in RS_INSTANCES:
        tag = f"rs/{inst[0]}-{inst[1]}"
        seq = rs_sequence(inst)
        names = [(o["op"], o.get("ncols")) for o in seq]
        for a, b in zip(names, names[1:]):
            r.add(f"{tag}:{a[0]}->{b[0]}")
            if a[0] == b[0] == "dev" and a[1] > 1 and b[1] == 1:
                r.add(f"{tag}:matrix->vector")
        if any(o["op"] == "stream" and o["hist"] for o in seq):
            r.add(f"{tag}:stream-history")
        if any(o["op"] == "refuse" for o in seq):
            r.add("refuse:resample")
    hs = [arb_touch(o).get("hist") for o in arb_sequence()]
    hs = [h for h in hs if h is not None]
    for a, b in zip(hs, hs[1:]):
        if a != b:
            r.add("arb:hist->plain" if a else "arb:plain->hist")
    r |= {"fir-filter:reset", "fir-filter:setphase", "fir-filter:device"}      # test_fir_filter_reuse runs these
    for inst in FIR_INSTANCES:
        tag = f"fir/{inst[0].name}"
        seq = fir_sequence(inst)
        cols = [o["ncols"] for o in seq if o["op"] != "refuse"]
        for a, b in zip(cols, cols[1:]):
            r.add(f"{tag}:cols{a}->{b}")
        forms = [o["op"] for o in seq]
        for a, b in zip(forms, forms[1:]):
            if a.startswith("host") != b.startswith("host") and "refuse" not in (a, b):
                r.add(f"{tag}:{'host->dev' if a.startswith('host') else 'dev->host'}")
            if a == "dev" and b == "state_dev":
                r.add(f"{tag}:stateless->stateful")
        _grow_shrink(f"{tag}:host", [fir_touch(inst, o).get("bytes") for o in seq], r)
        if "refuse" in forms:
            r.add("refuse:fir")
    seq = planless_sequence()
    model = lru_model(seq)
    keys = {k for o in seq if o["op"] in ("conv_fft", "conv_os", "hilbert", "per2") for k in planless_keys(o)}
    if len(keys) >= 40:
        r.add("planless:40-keys")
    first_keys = set(planless_keys(seq[0]))
    evicted_at = next((i for i, m in enumerate(model) if first_keys & set(m["evicted"])), None)
    if evicted_at is not None:
        r.add("planless:lru-evicts-first")
        if any(o.get("id") == seq[0]["id"] for o in seq[evicted_at + 1:]):
            r.add("planless:revisit-evicted")
    arena = [conv_fft_arena(o)[3] if o["op"] == "conv_fft" else None for o in seq]
    big = [i for i, o in enumerate(seq) if o.get("big")]
    if big:
        _grow_shrink("planless:arena", arena[big[0]:], r)
        if any(arena[i] > ARENA_KEEP for i in big):
            r.add("planless:arena-trim")
    if sum(o["op"] == "set_budget" for o in seq) >= 2 and seq[[o["op"] for o in seq].index("set_budget")]["budget"] != \
            DEFAULT_BUDGET:
        r.add("planless:budget-change-restore")
    if any(o["op"] == "refuse" for o in seq):
        r.add("refuse:planless")
    return r


def required_transitions():
    req = set()
    for inst in OS_INSTANCES:
        t = f"os/{_os_id(inst)}"
        req |= {f"{t}:dev70->dev1", f"{t}:range", f"{t}:state+si", f"{t}:state-si", f"{t}:host-chunked->host-short",
                f"{t}:pipe:reuse-smaller", f"{t}:stateful->stateless"}
    req |= {"os-cache:evict", "os-cache:revisit-evicted", "os-cache:host-dev-shared"}
    for wp in WELCH_PLANS:
        t = f"welch/{_wid(wp)}"
        req |= {f"{t}:welch-class-alternates", f"{t}:acc->batch->acc", f"{t}:filt_welch-lengths", f"{t}:host_welch-lengths"}
    fw = f"welch/{_wid(WELCH_PLANS[0])}"
    req |= {f"{fw}:batch-in-channel-groups", f"{fw}:bpartial:reuse-smaller", f"{fw}:pin->call", f"{fw}:unpin->call"}
    for sp in STFT_PLANS:
        t = f"stft/{_wid(sp)}"
        req |= {f"{t}:oneshot->stream", f"{t}:stream->oneshot", f"{t}:raw-psd-acc", f"{t}:seam"}
    req.add("stft:w1k")
    fused_mt, cufft_mt = (f"mt/{_wid(m)}" for m in MT_PLANS)
    req |= {f"{fused_mt}:bpartial:grow", f"{fused_mt}:bpartial:reuse-smaller", f"{cufft_mt}:tmp:grow",
            f"{cufft_mt}:tmp:reuse-smaller"}
    for m in MT_PLANS:
        req |= {f"mt/{_wid(m)}:pgram-batch->vector", f"mt/{_wid(m)}:spec-batch->vector", f"mt/{_wid(m)}:plain-batch-between"}
    for inst in RS_INSTANCES:
        t = f"rs/{inst[0]}-{inst[1]}"
        req |= {f"{t}:matrix->vector", f"{t}:dev->range", f"{t}:range->stream", f"{t}:stream->host", f"{t}:stream-history"}
    req |= {"fir-filter:reset", "fir-filter:setphase", "fir-filter:device", "arb:hist->plain", "arb:plain->hist"}
    for inst in FIR_INSTANCES:
        t = f"fir/{inst[0].name}"
        req |= {f"{t}:cols70->1", f"{t}:cols1->3", f"{t}:stateless->stateful", f"{t}:host->dev", f"{t}:dev->host",
                f"{t}:host:reuse-smaller"}
    req |= {"planless:40-keys", "planless:lru-evicts-first", "planless:revisit-evicted", "planless:arena:grow",
            "planless:arena:reuse-smaller", "planless:arena:regrow", "planless:arena-trim", "planless:budget-change-restore"}
    req |= {f"refuse:{k}" for k in ("os", "spec", "stft", "mt", "resample", "fir", "planless")}
    return req


# =============================================================================== CPU tests

def test_sequences_are_seeded_and_deterministic():
    for build in (lambda: [os_sequence(i) for i in OS_INSTANCES], front_sequence,
                  lambda: [welch_sequence(w) for w in WELCH_PLANS], lambda: [stft_sequence(s) for s in STFT_PLANS],
                  lambda: [mt_sequence(m) for m in MT_PLANS], lambda: [rs_sequence(i) for i in RS_INSTANCES],
                  arb_sequence, lambda: [fir_sequence(i) for i in FIR_INSTANCES], planless_sequence):
        assert build() == build()
    a, b = _rng("os", 3, 1).integers(0, 1 << 30, 4), _rng("os", 3, 1).integers(0, 1 << 30, 4)
    assert np.array_equal(a, b) and not np.array_equal(a, _rng("os", 3, 2).integers(0, 1 << 30, 4))


def test_restated_state():
    # Welch: an accumulation writes its rows on the first launch after begin and adds on every later one, in whichever
    # alignment class each launch runs
    wp = WELCH_PLANS[0]
    acc = next(o for o in welch_sequence(wp) if o["op"] == "acc" and o["batch"])
    t = welch_touch(wp, acc)
    assert [m for _, _, m in t["launches"]] == ["write"] + ["add"] * (len(t["launches"]) - 1)
    assert {c for _, c, _ in t["launches"]} == {0, 1}
    assert t["batch"]["groups"] == 2 and t["batch"]["bpartial"] == WELCH_BATCH_SCRATCH
    assert welch_class(F32, 2048, 4096, 1) == 0 and welch_class(F32, 2048, 4096, 4) == 1
    assert welch_class(F32, 250, 1000, 0) == 0                         # hop * 4 bytes is not a multiple of 16
    # plan-less keys: a real FFT conv asks for two plans, hilbert two, a 2-D periodogram one (shared by calls of one
    # transform size: the full and radial forms, an overlap-save block of the same dims)
    cyc = planless_cycle()
    keys = [k for o in cyc for k in planless_keys(o)]
    assert len(set(keys)) >= 40
    assert planless_keys(cyc[-4])[0] == planless_keys(cyc[-5])[0]
    assert planless_keys(dict(op="per2", nfft=(64, 40)))[0][1] == (40, 64)
    # the small budget batches two blocks at a time, the default all 6 x 8 (save_blocksize 52 x 12 of 312 x 94 outputs)
    op = dict(op="conv_os", us=(300, 90), vs=(13, 5), nffts=(64, 16))
    assert conv_os_batch(op, 2 * (64 * 16 * 4 + 33 * 16 * 8)) == 2 and conv_os_batch(op, DEFAULT_BUDGET) == 6 * 8
    # the LRU model evicts the least recently used key
    m = lru_model([dict(op="hilbert", n=i + 2, ncols=1) for i in range(17)] + [dict(op="hilbert", n=2, ncols=1)], cap=32)
    assert m[16]["evicted"] == planless_keys(dict(op="hilbert", n=2, ncols=1)) and m[17]["hits"] == []
    # the arena: the large call's slots stay (<= 256 MiB), the trimmed one's do not
    arena = [o for o in planless_sequence() if o.get("big")]
    assert max(conv_fft_arena(arena[0]).values()) <= ARENA_KEEP < min(conv_fft_arena(arena[1]).values())
    # overlap-save: the long host call is chunked, the short one is not
    for inst in OS_INSTANCES:
        hosts = [os_touch(inst, o) for o in os_sequence(inst) if o["op"] == "host"]
        assert [h["chunked"] for h in hosts] == [True, False]
    # the front-end cache evicts the first taps when the ninth set arrives, and the revisit misses
    model = front_cache_model(front_sequence())
    assert [ev for _, ev in model].count(0) == 1 and model[-2] == (False, 1)


def test_sequences_reach_every_transition():
    reached, required = reached_transitions(), required_transitions()
    assert required <= reached, sorted(required - reached)


# =============================================================================== GPU harness

@pytest.fixture(scope="module")
def dsp():
    return pytest.importorskip("dspb200")


def _rng(name, *k):
    return np.random.default_rng([sum(map(ord, name)), len(name)] + [int(v) for v in k])


class Bufs:
    """The guarded device buffers of one call, allocated once, so that the call on the sequence's plan and on the fresh plan
    read and write the same addresses.  Inputs between sentinels must come back unchanged; outputs between NaN cells are
    reset before every run."""

    def __init__(self):
        self.ins, self.outs = [], []

    def inp(self, dt, data, rng, off=0):
        g = kp.Guarded(dt, data.size, rng, data, offset=off)
        self.ins.append(g)
        return g

    def out(self, dt, n, prefill=None, off=0):
        g = kp.Guarded(dt, n, data=prefill, offset=off)
        self.outs.append(g)
        return g

    def reset(self):
        for g in self.outs:
            g.buf.copy_from_host(g.host)

    def results(self):
        from dspb200 import device
        device.sync()
        for g in self.ins:
            d = g.data()
            assert np.array_equal(d, g.host[g.lo:g.lo + g.n]), "a call wrote its input"
        return [g.data() for g in self.outs]


class Step:
    """One call.  run(plans) issues it and returns its outputs; oracle(fresh_plans) is the same call on fresh plans (default:
    run); check(outputs) compares with the integer or float64 reference; after(plans, fresh) compares what the plans report;
    solo: a call with no fresh twin (a refusal, which must fail with EINVALID before any launch, or a pin)."""

    def __init__(self, label, run, check=None, oracle=None, solo=False, after=None):
        self.label, self.run, self.check, self.oracle, self.solo, self.after = label, run, check, oracle, solo, after


def _close(plans):
    for p in plans:
        if hasattr(p, "close"):
            p.close()


def run_sequence(make, steps, prepare_fresh=None):
    """The steps on one set of plans; after each, the same call on freshly made plans must give the same bits."""
    from dspb200 import device
    plans = make()
    try:
        for st in steps:
            got = st.run(plans)
            if st.solo:
                continue
            fresh = make()
            try:
                if prepare_fresh is not None:
                    prepare_fresh(fresh)
                ref = (st.oracle or st.run)(fresh)
                if st.after is not None:
                    st.after(plans, fresh)
            finally:
                _close(fresh)
            assert len(got) == len(ref), st.label
            for i, (a, b) in enumerate(zip(got, ref)):
                assert same_bits(np.asarray(a), np.asarray(b)), (st.label, i, "differs from a fresh plan")
            if st.check is not None:
                st.check(got)
    finally:
        _close(plans)
        device.empty_cache()


def refused(dsp, fn):
    """fn must raise EINVALID and launch nothing."""
    n0 = dsp.launch_count()
    with pytest.raises(dsp._lib.DSPB200Error) as e:
        fn()
    assert e.value.code == dsp._lib.EINVALID, e.value
    assert dsp.launch_count() == n0
    return []


# =============================================================================== GPU: 1. overlap-save plans

def _os_state_ref(x, v, si):
    """Stateful overlap-save per column: full = conv(v, x), full[:nv-1] += si, out = full[:nx], si_out = the rest."""
    nx, ns = x.shape[0], v.size - 1
    full = osk.exact_conv(x, v)
    if si is not None:
        full[:ns] += si
    return full[:nx], full[nx:nx + ns]


def os_steps(dsp, inst, rng):
    dt, N, nv = inst
    f64 = dt in (F64, np.dtype(np.complex128))
    taps = osk.int_taps(rng, nv, dt)
    L = N - nv + 1
    steps = []
    for i, op in enumerate(os_sequence(inst)):
        r = _rng("os", N, nv, i)
        b = Bufs()
        label = (_os_id(inst), i, op["op"])
        if op["op"] == "dev":
            u = osk.int_signal(r, (op["nu"], op["ncols"]), dt)
            gu, go = b.inp(dt, u, r, op["off"]), b.out(dt, op["nout"] * op["ncols"], off=op["off"])

            def run(plans, b=b, gu=gu, go=go, op=op):
                b.reset()
                plans[0].exec_dev(gu.ptr, op["nu"], op["ncols"], go.ptr, op["nout"], 0)
                return [x.reshape(op["nout"], op["ncols"], order="F") for x in b.results()]

            def check(got, label=label, u=u, op=op):
                osk.check_exact(got[0], osk.exact_conv(u, taps, op["nout"]), f64, u.shape[0] + nv - 1, label)
        elif op["op"] == "range":
            u = osk.int_signal(r, op["nu"], dt)
            gu, go = b.inp(dt, u, r), b.out(dt, op["count"])

            def run(plans, b=b, gu=gu, go=go, op=op):
                b.reset()
                plans[0].exec_range_dev(gu.ptr, op["u_begin"], op["nu"], go.ptr, op["out_begin"], op["count"], 0)
                return b.results()

            def check(got, label=label, u=u, op=op):
                full = osk.exact_conv(u, taps)
                m = np.arange(op["out_begin"], op["out_begin"] + op["count"]) - op["u_begin"]
                want = np.where((m >= 0) & (m < full.size), full[np.clip(m, 0, full.size - 1)], 0)
                osk.check_exact(got[0], want, f64, what=label)
        elif op["op"] == "state":
            nx, nc, ns = op["nx"], op["ncols"], nv - 1
            x = osk.int_signal(r, (nx, nc), dt)
            si = osk.int_signal(r, (ns, nc), dt) if op["si"] else None
            gx = b.inp(dt, x, r)
            gs = b.inp(dt, si, r) if op["si"] else None
            go, gso = b.out(dt, nx * nc), b.out(dt, ns * nc)

            def run(plans, b=b, gx=gx, gs=gs, go=go, gso=gso, nx=nx, nc=nc):
                b.reset()
                plans[0].exec_state_dev(gx.ptr, nx, nc, gs.ptr if gs else None, gso.ptr, go.ptr, 0)
                y, s = b.results()
                return [y.reshape(nx, nc, order="F"), s.reshape(ns, nc, order="F")]

            def check(got, label=label, x=x, si=si):
                y, s = _os_state_ref(x, taps, si)
                osk.check_exact(got[0], y, f64, what=label)
                osk.check_exact(got[1], s, f64, what=label)
        elif op["op"] == "host":
            u = np.asfortranarray(osk.int_signal(r, (op["nu"], op["ncols"]), dt))

            def run(plans, u=u, op=op):
                out = np.full((op["nout"], op["ncols"]), np.nan, dtype=dt, order="F")
                plans[0].exec(u, out, op["nu"], op["ncols"], op["nout"])
                return [out]

            def check(got, label=label, u=u, op=op):
                osk.check_exact(got[0], osk.exact_conv(u, taps, op["nout"]), f64, what=label)
        else:
            x = osk.int_signal(r, (L, 2), dt)
            gx, gs, go = b.inp(dt, x, r), b.inp(dt, osk.int_signal(r, (nv - 1, 2), dt), r), b.out(dt, 2 * L)
            steps.append(Step(label, lambda plans, gx=gx, gs=gs, go=go: refused(
                dsp, lambda: plans[0].exec_state_dev(gx.ptr, L, 2, gs.ptr, gs.ptr, go.ptr, 0)), solo=True))
            continue
        steps.append(Step(label, run, check))
    return taps, steps


@pytest.mark.gpu
@pytest.mark.parametrize("inst", OS_INSTANCES, ids=[_os_id(i) for i in OS_INSTANCES])
def test_os_plan_sequence(dsp, inst):
    dt, N, nv = inst
    taps, steps = os_steps(dsp, inst, _rng("os-taps", N, nv))
    nfft = 0 if osk.os_fused_ok(N, nv, dt == F64) and osk.auto_nfft(nv, dt == F64) == N else N

    def make():
        p = dsp._lib.OsPlan(taps, nfft)
        assert p.nfft == N and p.fused == osk.os_fused_ok(N, nv, dt == F64)
        return [p]

    run_sequence(make, steps)


@pytest.mark.gpu
def test_front_end_os_plan_cache(dsp):
    """fftfilt / conv share _OS_PLANS across host and device arrays, lengths and column counts; a ninth set of taps evicts
    the first, whose next call runs on a new plan and must give the bits of the first call."""
    from dspb200 import dspbase, device
    from dspb200.device import to_device
    saved = dict(dspbase._OS_PLANS)
    dspbase._OS_PLANS.clear()
    try:
        tapsets = [osk.int_taps(_rng("front", t), 150 + 7 * t, F32) for t in range(FRONT_TAPS)]
        first, model = {}, front_cache_model(front_sequence())
        for i, op in enumerate(front_sequence()):
            r = _rng("front-x", {12: 0, 13: 1}.get(i, i))            # the last two revisit the first two calls
            v = tapsets[op["taps"]]
            before = dict(dspbase._OS_PLANS)
            if op["op"].startswith("fftfilt"):
                x = osk.int_signal(r, (op["nx"], op["ncols"]), F32)
                y = dsp.fftfilt(v, to_device(np.asfortranarray(x))).to_host() if op["op"] == "fftfilt_dev" else \
                    dsp.fftfilt(v, x)
                want = osk.exact_conv(x, v, op["nx"])
            else:
                u = osk.int_signal(r, op["nu"], F32)
                y = dsp.conv(to_device(u), v).to_host() if op["op"] == "conv_dev" else \
                    dsp.conv(u, v, algorithm="fft_overlapsave")
                want = osk.exact_conv(u, v)
            device.sync()
            osk.check_exact(np.asarray(y), want, False, what=(i, op))
            hit, ev = model[i]
            assert (len(dspbase._OS_PLANS) == len(before)) == (hit or ev is not None), (i, op)
            key = (op["op"], op["taps"])
            if key in first:                         # a revisit (after the eviction for taps 0) equals its first run
                assert same_bits(np.asarray(y), first[key]), (i, op)
            first.setdefault(key, np.asarray(y))
            # the cached plan's result equals a fresh plan's on the same data
            if op["op"] == "fftfilt_host":
                p = dsp._lib.OsPlan(v, 0)
                try:
                    xr = np.asfortranarray(x)
                    out = np.empty_like(xr)
                    p.exec(xr, out, op["nx"], op["ncols"], op["nx"])
                finally:
                    p.close()
                assert same_bits(np.asarray(y).reshape(out.shape, order="F"), out), (i, op)
        assert sum(ev == 0 for _, ev in model) == 1
    finally:
        for p in dspbase._OS_PLANS.values():
            p.close()
        dspbase._OS_PLANS.clear()
        dspbase._OS_PLANS.update(saved)
        device.empty_cache()


# =============================================================================== GPU: 2. Welch

class SpecCtx:
    """Pins carried over to the fresh plans (a pinned plan's fresh twin is pinned the same way)."""

    def __init__(self):
        self.pins = {}

    def prepare(self, fresh):
        for batched, pin in self.pins.items():
            fresh[0].pin_welch(batched, *pin)


def _welch_ref(x, n, hop, N, w, onesided=True):
    return kp.ref_segments(x, n, hop, N, w)


def welch_steps(dsp, wp, ctx):
    dt, N, hop = wp
    n, u = N, kp.eps(dt)
    w = kp.window_of("hann", n, None)
    norm2 = kp.norm2_of(w, n)
    steps = []
    taps = kp.signal(_rng("fw-taps", N), 65, dt) * 0.1

    pins = {}

    def cfg_after(form, cls):
        """After a call: the configuration the sequence's plan reports for the form and class the call used equals the
        fresh plan's, and a pinned instance is the one that ran (the others run MODE 0, G = 1) (fused sizes)."""
        pin = pins.get(form)

        def after(plans, fresh):
            if not kp.fused_size_ok(N, False):
                return
            got = plans[0].welch_config(form, cls)
            assert got == fresh[0].welch_config(form, cls) and got[1] > 0, (form, cls, got)
            if pin is not None:
                want = (pin[0], pin[1]) if cls else (0, 1)
                assert got[:2] == want and (form == 1 or got[2] == pin[2]), (form, cls, got, pin)
        return after

    for i, op in enumerate(welch_sequence(wp)):
        if op["op"] == "pin":
            if op["mode"] < 0:
                pins.pop(op["batched"], None)
            else:
                pins[op["batched"]] = (op["mode"], op["groups"], op["vctas"])
        r = _rng("welch", N, i)
        b = Bufs()
        label = (_wid(wp), i, op["op"])
        if op["op"] == "welch":
            k = op["k"]
            length = (k - 1) * hop + n
            x = kp.signal(r, length, dt)
            gx, go = b.inp(dt, x, r, op["off"]), b.out(F32, N // 2 + 1)

            def run(plans, b=b, gx=gx, go=go, length=length, k=k):
                b.reset()
                plans[0].welch_dev(gx.ptr, length, k * norm2, go.ptr, 0)
                return b.results()

            def check(got, label=label, x=x, k=k):
                X, en = _welch_ref(x, n, hop, N, w)
                kp.check_welch(got[0], X, en, N, True, k * norm2, u, cdiv(k, 2), label)

            steps.append(Step(label, run, check, after=cfg_after(0, welch_class(dt, hop, n, op["off"]))))
        elif op["op"] in ("acc", "refuse"):
            k = op["k"]
            length = (k - 1) * hop + n
            x = kp.signal(r, length, dt)
            pieces = []
            for bb, e, off in op["chunks"] + op["rest"]:
                lo, hi = bb * hop, (e - 1) * hop + n
                pieces.append((b.inp(dt, x[lo:hi], r, off), hi - lo, lo, bb, e))
            nfirst = len(op["chunks"])
            go = b.out(F32, N // 2 + 1)
            bt = op.get("batch")
            blen = xb = gb = gbo = None
            if bt:
                blen = (bt["k"] - 1) * hop + n
                xb = kp.signal(r, (blen, bt["nchan"]), dt)
                gb, gbo = b.inp(dt, xb, r, bt["off"]), b.out(F32, (N // 2 + 1) * bt["nchan"])
            if op["op"] == "refuse":
                def run(plans, refuse=True, b=b, pieces=pieces, go=go, nfirst=nfirst, k=k):
                    """An open accumulation, a refused accumulate in its middle (the oracle: the same without it)."""
                    b.reset()
                    p = plans[0]
                    p.welch_begin_dev(0)
                    for g, ln, lo, bb, e in pieces[:nfirst]:
                        p.welch_accumulate_dev(g.ptr, ln, lo, bb, e, 0)
                    if refuse:
                        refused(dsp, lambda: p.welch_accumulate_dev(pieces[0][0].ptr, pieces[0][1], INDEX_LIMIT, 0, 1, 0))
                    for g, ln, lo, bb, e in pieces[nfirst:]:
                        p.welch_accumulate_dev(g.ptr, ln, lo, bb, e, 0)
                    p.welch_finalize_dev(k * norm2, go.ptr, 0)
                    return b.results()

                def oracle(fresh, run=run):
                    return run(fresh, False)
            else:
                def seq_run(plans, with_batch, b=b, pieces=pieces, go=go, nfirst=nfirst, k=k, bt=bt, gb=gb, gbo=gbo,
                            blen=blen):
                    b.reset()
                    p = plans[0]
                    p.welch_begin_dev(0)
                    for g, ln, lo, bb, e in pieces[:nfirst]:
                        p.welch_accumulate_dev(g.ptr, ln, lo, bb, e, 0)
                    if bt and with_batch:
                        p.welch_batch_dev(gb.ptr, blen, bt["nchan"], bt["k"] * norm2, gbo.ptr, 0)
                    for g, ln, lo, bb, e in pieces[nfirst:]:
                        p.welch_accumulate_dev(g.ptr, ln, lo, bb, e, 0)
                    p.welch_finalize_dev(k * norm2, go.ptr, 0)
                    res = b.results()
                    return res if with_batch else res[:1]

                def run(plans, seq_run=seq_run):
                    return seq_run(plans, True)

                def oracle(fresh, seq_run=seq_run, bt=bt, b=b, gb=gb, gbo=gbo, blen=blen):
                    """The accumulation alone on a fresh plan; the batch on another fresh plan."""
                    res = seq_run(fresh, False)
                    if not bt:
                        return res
                    other = welch_make(dsp, wp)
                    try:
                        ctx.prepare(other)
                        b.reset()
                        other[0].welch_batch_dev(gb.ptr, blen, bt["nchan"], bt["k"] * norm2, gbo.ptr, 0)
                        return res + b.results()[1:]
                    finally:
                        _close(other)

            def check(got, label=label, x=x, k=k, bt=bt, xb=xb):
                X, en = _welch_ref(x, n, hop, N, w)
                kp.check_welch(got[0], X, en, N, True, k * norm2, u, cdiv(k, 2), label)
                if bt:
                    P = got[1].reshape(N // 2 + 1, bt["nchan"], order="F")
                    for c in {0, bt["nchan"] // 2, bt["nchan"] - 1}:
                        Xc, ec = _welch_ref(xb[:, c], n, hop, N, w)
                        kp.check_welch(P[:, c], Xc, ec, N, True, bt["k"] * norm2, u, cdiv(bt["k"], 2), (label, c))

            steps.append(Step(label, run, check, oracle=oracle))
        elif op["op"] == "batch":
            length = (op["k"] - 1) * hop + n
            xb = kp.signal(r, (length, op["nchan"]), dt)
            gb, go = b.inp(dt, xb, r, op["off"]), b.out(F32, (N // 2 + 1) * op["nchan"])

            def run(plans, b=b, gb=gb, go=go, length=length, op=op):
                b.reset()
                plans[0].welch_batch_dev(gb.ptr, length, op["nchan"], op["k"] * norm2, go.ptr, 0)
                return b.results()

            def check(got, label=label, xb=xb, op=op):
                P = got[0].reshape(N // 2 + 1, op["nchan"], order="F")
                for c in range(op["nchan"]):
                    X, en = _welch_ref(xb[:, c], n, hop, N, w)
                    kp.check_welch(P[:, c], X, en, N, True, op["k"] * norm2, u, cdiv(op["k"], 2), (label, c))

            cls = welch_batch_class(dt, hop, n, op["off"], length, op["nchan"])
            steps.append(Step(label, run, check, after=cfg_after(1, cls)))
        elif op["op"] == "filt_welch":
            k = op["k"]
            length = (k - 1) * hop + n
            x = kp.signal(r, length, dt)

            def run(plans, x=x, k=k):
                out = np.full(N // 2 + 1, np.nan, dtype=F32)
                plans[0].filt_welch_ptr(plans[1], dsp._lib.ptr(x), x.size, k * norm2, dsp._lib.ptr(out))
                return [out]

            def check(got, label=label, x=x, k=k):
                y = np.convolve(x.astype(np.float64), taps.astype(np.float64))[:x.size]
                X, en = _welch_ref(y, n, hop, N, w)
                b_, mult = kp.bins_and_mult(N, True)
                want = np.mean(np.abs(X) ** 2, axis=0)[b_] * mult / (k * norm2 / k)
                assert np.abs(got[0] - want).max() <= 1e-4 * want.max(), label

            steps.append(Step(label, run, check))
        elif op["op"] == "host_welch":
            k = op["k"]
            x = kp.signal(r, (k - 1) * hop + n, dt)

            def run(plans, x=x, k=k):
                out = np.full(N // 2 + 1, np.nan, dtype=F32)
                plans[0].welch(x, k * norm2, out)
                return [out]

            def check(got, label=label, x=x, k=k):
                X, en = _welch_ref(x, n, hop, N, w)
                kp.check_welch(got[0], X, en, N, True, k * norm2, u, cdiv(min(k, kp.host_chunk_segs(4, hop, k)), 2), label)

            steps.append(Step(label, run, check))
        elif op["op"] == "pin":
            def run(plans, op=op):
                p = plans[0]
                p.pin_welch(op["batched"], op["mode"], op["groups"], op["vctas"])
                if op["mode"] < 0:
                    ctx.pins.pop(op["batched"], None)
                else:
                    ctx.pins[op["batched"]] = (op["mode"], op["groups"], op["vctas"])
                for cls in (0, 1):                   # pinning or unpinning forgets the last call's configuration
                    assert p.welch_config(op["batched"], cls) == (-1, 0, 0)
                return []

            steps.append(Step(label, run, solo=True))            # changes no output: the calls after it are compared
    return steps


def welch_make(dsp, wp):
    dt, N, hop = wp
    spec = dsp._lib.SpecPlan(dt, N, N - hop, N, True, kp.window_of("hann", N, None))
    assert spec.fused == kp.fused_size_ok(N, False)
    os_ = dsp._lib.OsPlan(kp.signal(_rng("fw-taps", N), 65, dt) * 0.1, 0)
    return [spec, os_]


@pytest.mark.gpu
@pytest.mark.parametrize("wp", WELCH_PLANS, ids=[_wid(w) for w in WELCH_PLANS])
def test_welch_plan_sequence(dsp, wp):
    ctx = SpecCtx()
    steps = welch_steps(dsp, wp, ctx)
    run_sequence(lambda: welch_make(dsp, wp), steps, ctx.prepare)


# =============================================================================== GPU: 3. STFT

def stft_steps(dsp, sp):
    dt, N, hop = sp
    n, u = N, kp.eps(dt)
    cplx = dt.kind == "c"
    onesided = not cplx
    nout = N // 2 + 1 if onesided else N
    w = kp.window_of("hann", n, None)
    r_psd = kp.norm2_of(w, n)
    cdt = C64
    steps = []
    for i, op in enumerate(stft_sequence(sp)):
        r = _rng("stft", N, i)
        b = Bufs()
        label = (_wid(sp), i, op["op"])
        if op["op"] in ("stft", "stft_acc"):
            k, nc = op["k"], op["nchan"]
            length = (k - 1) * hop + n
            x = kp.signal(r, (length, nc), dt)
            gx = b.inp(dt, x, r)
            psd = 1 if op["op"] == "stft_acc" else op["psd"]
            go = b.out(F32 if psd else cdt, nout * k * nc)
            pre = (r.random(nout * k * nc) * 4).astype(F32) if op["op"] == "stft_acc" else None
            ga = b.out(F32, nout * k * nc, prefill=pre) if pre is not None else None

            def run(plans, b=b, gx=gx, go=go, ga=ga, length=length, nc=nc, psd=psd):
                b.reset()
                lib = dsp._lib
                lib.check(lib.lib.dspb200_stft_exec_dev(plans[0].handle, gx.ptr, length, nc, r_psd, psd, go.ptr, None))
                if ga is not None:
                    lib.check(lib.lib.dspb200_stft_exec_dev(plans[0].handle, gx.ptr, length, nc, r_psd, 3, ga.ptr, None))
                return b.results()

            def check(got, label=label, x=x, k=k, nc=nc, psd=psd, pre=pre):
                refs = [kp.ref_segments(x[:, c], n, hop, N, w) for c in range(nc)]
                X, en = np.concatenate([a for a, _ in refs]), np.concatenate([e for _, e in refs])
                Y = got[0].reshape(nout, k * nc, order="F")
                if psd:
                    kp.check_stft_psd(Y, X, en, N, onesided, r_psd, u, label)
                else:
                    kp.check_stft_raw(Y, X, en, N, onesided, u, label)
                if pre is not None:
                    assert same_bits(got[1], (pre + got[0]).astype(F32)), label

            steps.append(Step(label, run, check))
        elif op["op"] == "stream":
            nc, nh, nseg = op["nchan"], op["nhist"], op["nseg"]
            nx = (nseg - 1) * hop + n - nh + op["extra"]
            ldh = N
            hist = kp.signal(r, (ldh, nc), dt)
            x = kp.signal(r, (nx, nc), dt)
            gh = b.inp(dt, hist, r) if nh else None
            gx = b.inp(dt, x, r)
            newh = nh + nx - nseg * hop
            gho = b.out(dt, ldh * nc)
            go = b.out(F32 if op["psd"] else cdt, nout * nseg * nc)

            def run(plans, b=b, gh=gh, gx=gx, gho=gho, go=go, nh=nh, nx=nx, nc=nc, nseg=nseg, psd=op["psd"], newh=newh):
                b.reset()
                plans[0].stft_stream_dev(gh.ptr if gh else None, nh, gho.ptr, ldh, gx.ptr, nx, nc, nseg, r_psd, psd, go.ptr,
                                         nseg, 0)
                hout, y = b.results()
                return [hout.reshape(ldh, nc, order="F")[:newh], y]

            def check(got, label=label, hist=hist, x=x, nh=nh, nc=nc, nseg=nseg, psd=op["psd"], newh=newh):
                Y = got[1].reshape(nout, nseg * nc, order="F")
                Xs, es = [], []
                for c in range(nc):
                    v = np.concatenate([hist[:nh, c], x[:, c]])
                    assert same_bits(got[0][:, c], v[nseg * hop:]), (label, "new history")
                    X, en = kp.ref_segments(v[:(nseg - 1) * hop + n], n, hop, N, w)
                    Xs.append(X)
                    es.append(en)
                X, en = np.concatenate(Xs), np.concatenate(es)
                if psd:
                    kp.check_stft_psd(Y, X, en, N, onesided, r_psd, u, label)
                else:
                    kp.check_stft_raw(Y, X, en, N, onesided, u, label)

            steps.append(Step(label, run, check))
        else:
            nx = 3 * hop + n
            x = kp.signal(r, (nx, 1), dt)
            gx, go = b.inp(dt, x, r), b.out(cdt, nout * 4)
            steps.append(Step(label, lambda plans, gx=gx, go=go, nx=nx: refused(dsp, lambda: plans[0].stft_stream_dev(
                None, 0, gx.ptr, N, gx.ptr, nx, 1, 4, r_psd, 0, go.ptr, 4, 0)), solo=True))
    return steps


@pytest.mark.gpu
@pytest.mark.parametrize("sp", STFT_PLANS, ids=[_wid(s) for s in STFT_PLANS])
def test_stft_plan_sequence(dsp, sp):
    dt, N, hop = sp

    def make():
        p = dsp._lib.SpecPlan(dt, N, N - hop, N, dt.kind != "c", kp.window_of("hann", N, None))
        assert p.fused
        return [p]

    run_sequence(make, stft_steps(dsp, sp))


# =============================================================================== GPU: 4. multitaper

def mt_steps(dsp, mp):
    dt, N, hop, nt = mp
    n, u = N, kp.eps(dt)
    nout = N // 2 + 1
    rows = kp._tapers(n, nt)
    w = kp.window_of("hann", n, None)
    norm2 = kp.norm2_of(w, n)
    steps = []
    for i, op in enumerate(mt_sequence(mp)):
        r = _rng("mt", N, i)
        b = Bufs()
        label = (_wid(mp), i, op["op"])
        if op["op"] == "pgram":
            nc = op["nchan"]
            x = kp.signal(r, (n, nc), dt)
            gx, go = b.inp(dt, x, r), b.out(F32, nout * nc)

            def run(plans, b=b, gx=gx, go=go, nc=nc):
                b.reset()
                if nc == 1:
                    plans[0].mt_pgram_dev(gx.ptr, n, go.ptr, 0)
                else:
                    plans[0].mt_pgram_batch_dev(gx.ptr, n, nc, go.ptr, 0)
                return b.results()

            def check(got, label=label, x=x, nc=nc):
                P = got[0].reshape(nout, nc, order="F")
                for c in {0, nc // 2, nc - 1}:
                    segs = [kp.ref_segments(x[:, c], n, n, N, rows[t]) for t in range(nt)]
                    X, en = np.concatenate([s[0] for s in segs]), np.concatenate([s[1] for s in segs])
                    kp.check_welch(P[:, c], X, en, N, True, 1.0, u, nt, (label, c))
        elif op["op"] == "spec":
            nc, k = op["nchan"], op["k"]
            length = (k - 1) * hop + n
            x = kp.signal(r, (length, nc), dt)
            gx, go = b.inp(dt, x, r), b.out(F32, nout * k * nc)

            def run(plans, b=b, gx=gx, go=go, nc=nc, length=length):
                b.reset()
                if nc == 1:
                    plans[0].mt_spectrogram_dev(gx.ptr, length, go.ptr, 0)
                else:
                    plans[0].mt_spectrogram_batch_dev(gx.ptr, length, nc, go.ptr, 0)
                return b.results()

            def check(got, label=label, x=x, nc=nc, k=k):
                Y = got[0].reshape(nout, k * nc, order="F")
                bins, mult = kp.bins_and_mult(N, True)
                for c in range(nc):
                    for j in range(k):
                        seg = x[j * hop:j * hop + n, c]
                        segs = [kp.ref_segments(seg, n, n, N, rows[t]) for t in range(nt)]
                        S = sum(np.abs(s[0][0, bins]) ** 2 for s in segs)
                        E = float(sum(s[1][0] for s in segs))
                        kp.check_power(Y[:, c * k + j], S, E, mult, 1.0, u, N, nt, (label, c, j))
        elif op["op"] == "plain_batch":
            nc, k = op["nchan"], op["k"]
            length = (k - 1) * hop + n
            x = kp.signal(r, (length, nc), dt)
            gx, go = b.inp(dt, x, r), b.out(F32, nout * nc)

            def run(plans, b=b, gx=gx, go=go, nc=nc, length=length, k=k):
                b.reset()
                plans[1].welch_batch_dev(gx.ptr, length, nc, k * norm2, go.ptr, 0)
                return b.results()

            def check(got, label=label, x=x, nc=nc, k=k):
                P = got[0].reshape(nout, nc, order="F")
                for c in (0, nc - 1):
                    X, en = kp.ref_segments(x[:, c], n, hop, N, w)
                    kp.check_welch(P[:, c], X, en, N, True, k * norm2, u, cdiv(k, 2), (label, c))
        else:
            x = kp.signal(r, (n + 1, 2), dt)
            gx, go = b.inp(dt, x, r), b.out(F32, nout * 2)
            steps.append(Step(label, lambda plans, gx=gx, go=go: refused(
                dsp, lambda: plans[0].mt_pgram_batch_dev(gx.ptr, n + 1, 2, go.ptr, 0)), solo=True))
            continue
        steps.append(Step(label, run, check))
    return steps


@pytest.mark.gpu
@pytest.mark.parametrize("mp", MT_PLANS, ids=[_wid(m) for m in MT_PLANS])
def test_mt_plan_sequence(dsp, mp):
    dt, N, hop, nt = mp

    def make():
        p = dsp._lib.MtPlan(dt, N, N - hop, N, True, kp._tapers(N, nt))
        q = dsp._lib.SpecPlan(dt, N, N - hop, N, True, kp.window_of("hann", N, None))
        assert p.fused == q.fused == kp.fused_size_ok(N, False)
        return [p, q]

    run_sequence(make, mt_steps(dsp, mp))


# =============================================================================== GPU: 5. resampling

def rs_steps(dsp, inst, h):
    I, D, hlen = inst
    tpp = cdiv(hlen, I)
    H = tpp - 1
    n0, phi0 = tpp // 2, 1
    steps = []
    for i, op in enumerate(rs_sequence(inst)):
        r = _rng("rs", I, D, i)
        b = Bufs()
        label = (inst, i, op["op"])
        if op["op"] == "dev":
            nx, nc = op["nx"], op["ncols"]
            nout = nx * I // D
            x = rk.int_signal(r, (nx, nc), F32)
            gx, go = b.inp(F32, x, r), b.out(F32, nout * nc)

            def run(plans, b=b, gx=gx, go=go, nx=nx, nc=nc, nout=nout):
                b.reset()
                plans[0].exec_dev(gx.ptr, nx, nc, n0, phi0, go.ptr, nout, 0)
                return [b.results()[0].reshape(nout, nc, order="F")]

            def check(got, label=label, x=x, nout=nout):
                assert np.array_equal(got[0], rk.polyphase_ref(x, h, I, D, n0, phi0, nout)), label
        elif op["op"] == "range":
            x = rk.int_signal(r, op["nloc"], F32)
            gx, go = b.inp(F32, x, r), b.out(F32, op["count"])

            def run(plans, b=b, gx=gx, go=go, op=op):
                b.reset()
                plans[0].exec_range_dev(gx.ptr, op["x_begin"], op["nloc"], n0, phi0, go.ptr, op["j_begin"], op["count"], 0)
                return b.results()

            def check(got, label=label, x=x, op=op):
                xv = np.concatenate([np.zeros(op["x_begin"], F32), x])
                want = rk.polyphase_ref(xv, h, I, D, n0, phi0, op["j_begin"] + op["count"])[op["j_begin"]:]
                assert np.array_equal(got[0], want), label
        elif op["op"] == "stream":
            nx, nc = op["nx"], op["ncols"]
            nout = nx * I // D - 1
            hist = rk.int_signal(r, (H, nc), F32) if op["hist"] else np.zeros((H, nc), F32)
            x = rk.int_signal(r, (nx, nc), F32)
            gh = b.inp(F32, hist, r) if op["hist"] else None
            gx, gho, go = b.inp(F32, x, r), b.out(F32, H * nc), b.out(F32, nout * nc)

            def run(plans, b=b, gh=gh, gx=gx, gho=gho, go=go, nx=nx, nc=nc, nout=nout):
                b.reset()
                plans[0].stream_exec_dev(gh.ptr if gh else None, gho.ptr, gx.ptr, nx, nc, 1, 0, go.ptr, nout, nout, 0)
                ho, y = b.results()
                return [ho.reshape(H, nc, order="F"), y.reshape(nout, nc, order="F")]

            def check(got, label=label, hist=hist, x=x, nout=nout):
                v = np.concatenate([hist, x])
                assert np.array_equal(got[0], v[v.shape[0] - H:]), label
                assert np.array_equal(got[1], rk.polyphase_ref(v, h, I, D, H, 0, nout)), label
        elif op["op"] == "host":
            nx, nc = op["nx"], op["ncols"]
            nout = nx * I // D
            x = np.asfortranarray(rk.int_signal(r, (nx, nc), F32))

            def run(plans, x=x, nx=nx, nc=nc, nout=nout):
                out = np.full((nout, nc), np.nan, dtype=F32, order="F")
                plans[0].exec(x, nx, nc, n0, phi0, out, nout)
                return [out]

            def check(got, label=label, x=x, nout=nout):
                assert np.array_equal(got[0], rk.polyphase_ref(x, h, I, D, n0, phi0, nout)), label
        else:
            x = rk.int_signal(r, 1000, F32)
            gx, go = b.inp(F32, x, r), b.out(F32, 10)
            steps.append(Step(label, lambda plans, gx=gx, go=go: refused(
                dsp, lambda: plans[0].exec_range_dev(gx.ptr, 0, 1000, n0, phi0, go.ptr, INDEX_LIMIT, 10, 0)), solo=True))
            continue
        steps.append(Step(label, run, check))
    return steps


@pytest.mark.gpu
@pytest.mark.parametrize("inst", RS_INSTANCES, ids=[f"{i[0]}-{i[1]}-h{i[2]}" for i in RS_INSTANCES])
def test_resample_plan_sequence(dsp, inst):
    I, D, hlen = inst
    h = rk.int_taps(_rng("rs-taps", I, D), hlen, F32)
    run_sequence(lambda: [dsp._lib.ResamplePlan(F32, h, I, D)], rs_steps(dsp, inst, h))


def arb_steps(dsp):
    nph, hlen, rate = ARB
    H = cdiv(hlen, nph) - 1
    acc0, delta = 0.3, nph / rate
    steps = []
    for i, op in enumerate(arb_sequence()):
        r = _rng("arb", i)
        b = Bufs()
        label = ("arb", i, op["op"])
        nx = op["nx"]
        nout = int(nx * rate) - 5
        if op["op"] == "stream":
            nc = op["ncols"]
            hist, x = kp.signal(r, (H, nc), F32), kp.signal(r, (nx, nc), F32)
            gh, gx, gho, go = b.inp(F32, hist, r), b.inp(F32, x, r), b.out(F32, H * nc), b.out(F32, nout * nc)

            def run(plans, b=b, gh=gh, gx=gx, gho=gho, go=go, nx=nx, nc=nc, nout=nout):
                b.reset()
                plans[0].stream_exec_dev(gh.ptr, gho.ptr, gx.ptr, nx, nc, 1, acc0, delta, go.ptr, nout, nout, 0)
                return b.results()
        elif op["op"] == "batch":
            nc, ldx = op["ncols"], nx + 3
            x = kp.signal(r, (ldx, nc), F32)
            gx, go = b.inp(F32, x, r), b.out(F32, nout * nc)

            def run(plans, b=b, gx=gx, go=go, nx=nx, nc=nc, ldx=ldx, nout=nout):
                b.reset()
                plans[0].exec_batch_dev(gx.ptr, nx, ldx, nc, 0, acc0, delta, go.ptr, nout, 0)
                return b.results()
        elif op["op"] == "plain":
            x = kp.signal(r, nx, F32)
            gx, go = b.inp(F32, x, r), b.out(F32, nout)

            def run(plans, b=b, gx=gx, go=go, nx=nx, nout=nout):
                b.reset()
                plans[0].exec_dev(gx.ptr, nx, 0, acc0, delta, go.ptr, nout, 0)
                return b.results()
        else:
            x = kp.signal(r, (nx, 1), F32)
            gx, gho, go = b.inp(F32, x, r), b.out(F32, H), b.out(F32, nout)
            steps.append(Step(label, lambda plans, gx=gx, gho=gho, go=go, nx=nx, nout=nout: refused(
                dsp, lambda: plans[0].stream_exec_dev(None, gho.ptr, gx.ptr, nx, 1, 1, acc0, delta, go.ptr, nout - 1, nout,
                                                      0)), solo=True))
            continue
        steps.append(Step(label, run))
    return steps


@pytest.mark.gpu
def test_resample_arb_plan_sequence(dsp):
    nph, hlen, rate = ARB
    h = kp.signal(_rng("arb-taps"), hlen, F32)
    run_sequence(lambda: [dsp._lib.ResampleArbPlan(F32, h, nph)], arb_steps(dsp))


@pytest.mark.gpu
def test_fir_filter_reuse(dsp):
    """FIRFilter keeps its plans across reset() and setphase(): a reset filter repeats its first outputs bit for bit, a
    chunked stream equals one call over the concatenation, and a phase set after earlier calls equals a fresh filter with
    that phase.  The same for a device filter on channel matrices."""
    from dspb200.filters import FIRFilter
    from dspb200.device import to_device
    h = rk.int_taps(_rng("firf"), 38, F32)
    ratio = Fraction(3, 2)
    r = _rng("firf-x")
    x1, x2, x3 = (rk.int_signal(r, n, F32) for n in (5001, 3337, 4003))
    f = FIRFilter(h, ratio)
    a1, a2 = f.filt(x1), f.filt(x2)
    assert same_bits(np.concatenate([a1, a2]), FIRFilter(h, ratio).filt(np.concatenate([x1, x2])))
    st = FIRFilter(h, ratio)._step(1, 1, 0.0, x1.size)
    assert np.array_equal(a1, rk.polyphase_ref(np.concatenate([np.zeros(f.history_len, F32), x1]), h, 3, 2, st.n0,
                                               st.phase0, st.nout))
    f.reset()
    assert same_bits(f.filt(x1), a1)
    f.setphase(0.7)
    c = f.filt(x3)
    g = FIRFilter(h, ratio)
    g.filt(x1)
    g.setphase(0.7)
    assert same_bits(c, g.filt(x3))
    # device filter, three channels
    X1, X2 = (np.asfortranarray(rk.int_signal(r, (n, 3), F32)) for n in (4001, 2503))
    fd = FIRFilter(h, ratio, device=True)
    d1 = fd.filt(to_device(X1)).to_host()
    d2 = fd.filt(to_device(X2)).to_host()
    fd.reset()
    assert same_bits(fd.filt(to_device(X1)).to_host(), d1)
    e = fd.filt(to_device(X2)).to_host()
    assert same_bits(e, d2)
    fd.setphase(0.7)
    e3 = fd.filt(to_device(X1)).to_host()
    gd = FIRFilter(h, ratio, device=True)
    gd.filt(to_device(X1))
    gd.filt(to_device(X2))
    gd.setphase(0.7)
    assert same_bits(gd.filt(to_device(X1)).to_host(), e3)
    for c in range(3):                                   # each channel of the device stream is the host filter's
        hf = FIRFilter(h, ratio)
        assert same_bits(np.concatenate([hf.filt(X1[:, c]), hf.filt(X2[:, c])]), np.concatenate([d1[:, c], d2[:, c]]))


# =============================================================================== GPU: 6. FIR plans

def fir_steps(dsp, inst, b_taps):
    dt, nb = inst
    f64 = dt == F64
    ns = nb - 1
    steps = []

    def ref(x, si=None):
        return _os_state_ref(x, b_taps, si)

    for i, op in enumerate(fir_sequence(inst)):
        r = _rng("fir", nb, i)
        bf = Bufs()
        label = (dt.name, i, op["op"])
        if op["op"] == "refuse":
            x = osk.int_signal(r, (1000, 2), dt)
            gx = bf.inp(dt, x, r)
            go = bf.out(dt, ns * 2)
            steps.append(Step(label, lambda plans, gx=gx, go=go: refused(
                dsp, lambda: plans[0].exec_state_dev(gx.ptr, 1000, 2, None, go.ptr, gx.ptr, 0)), solo=True))
            continue
        nx, nc = op["nx"], op["ncols"]
        x = np.asfortranarray(osk.int_signal(r, (nx, nc), dt))
        si = osk.int_signal(r, (ns, nc), dt) if op.get("si") else None
        if op["op"] == "dev":
            gx, go = bf.inp(dt, x, r), bf.out(dt, nx * nc)

            def run(plans, bf=bf, gx=gx, go=go, nx=nx, nc=nc):
                bf.reset()
                plans[0].exec_dev(gx.ptr, nx, nc, go.ptr, 0)
                return [bf.results()[0].reshape(nx, nc, order="F")]
        elif op["op"] == "state_dev":
            gx = bf.inp(dt, x, r)
            gs = bf.inp(dt, si, r) if si is not None else None
            go, gso = bf.out(dt, nx * nc), bf.out(dt, ns * nc)

            def run(plans, bf=bf, gx=gx, gs=gs, go=go, gso=gso, nx=nx, nc=nc):
                bf.reset()
                plans[0].exec_state_dev(gx.ptr, nx, nc, gs.ptr if gs else None, gso.ptr, go.ptr, 0)
                y, s = bf.results()
                return [y.reshape(nx, nc, order="F"), s.reshape(ns, nc, order="F")]
        elif op["op"] == "host":
            def run(plans, x=x):
                out = np.full(x.shape, np.nan, dtype=dt, order="F")
                plans[0].exec(x, out)
                return [out]
        else:
            sif = np.asfortranarray(si)

            def run(plans, x=x, sif=sif, nx=nx, nc=nc):
                out = np.full(x.shape, np.nan, dtype=dt, order="F")
                so = np.full((ns, nc), np.nan, dtype=dt, order="F")
                plans[0].exec_state(x, nx, nc, sif, so, out)
                return [out, so]

        def check(got, label=label, x=x, si=si, op=op):
            y, s = ref(x, si)
            osk.check_exact(got[0], y, f64, what=label)
            if op["op"] in ("state_dev", "host_state"):
                osk.check_exact(got[1], s, f64, what=label)
            assert np.array_equal(got[0], y), label           # time-domain FIR on integers: exact, not merely rounded

        steps.append(Step(label, run, check))
    return steps


@pytest.mark.gpu
@pytest.mark.parametrize("inst", FIR_INSTANCES, ids=[f"{i[0].name}-nb{i[1]}" for i in FIR_INSTANCES])
def test_fir_plan_sequence(dsp, inst):
    dt, nb = inst
    b_taps = osk.int_taps(_rng("fir-taps", nb), nb, dt)
    run_sequence(lambda: [dsp._lib.FirPlan(b_taps)], fir_steps(dsp, inst, b_taps))


# =============================================================================== GPU: 7. plan-less calls

def _planless_data(op):
    r = _rng("planless", *[v for k in ("us", "vs", "nffts", "shape", "nfft") for v in op.get(k, ())],
             op.get("n", 0), op.get("ncols", 0))
    if op["op"] in ("conv_fft", "conv_os"):
        return [osk.int_signal(r, op["us"], F32), osk.int_taps(r, int(np.prod(op["vs"])), F32).reshape(op["vs"])]
    if op["op"] == "hilbert":
        return [kp.signal(r, (op["n"], op["ncols"]), F32)]
    return [kp.signal(r, op["shape"], F32)]


def _planless_run(dsp, op, data, rng):
    """One plan-less device call into guarded buffers; returns its output."""
    L = dsp._lib
    b = Bufs()
    if op["op"] in ("conv_fft", "conv_os"):
        u, v = data
        gu, gv = b.inp(F32, u, rng), b.inp(F32, v, rng)
        so = tuple(a + c - 1 for a, c in zip(op["us"], op["vs"]))
        go = b.out(F32, int(np.prod(so)))
        L.conv_nd_dev(F32, op["us"], gu.ptr, op["vs"], gv.ptr, op["nffts"], go.ptr, op["op"] == "conv_os", 0)
        return b.results()[0].reshape(so, order="F")
    if op["op"] == "hilbert":
        x = data[0]
        gx, go = b.inp(F32, x, rng), b.out(C64, x.size)
        L.hilbert_dev(F32, gx.ptr, op["n"], op["ncols"], go.ptr, 0)
        return b.results()[0]
    s = data[0]
    f1, f2 = op["nfft"]
    nout = f1 * f2 if op["ptype"] == 0 else min(f1, f2) // 2 + 1
    gs, go = b.inp(F32, s, rng), b.out(F32, nout)
    L.periodogram2_dev(F32, gs.ptr, op["shape"], op["nfft"], _per2_r(op), op["ptype"], go.ptr, 0)
    return b.results()[0]


def _per2_r(op):
    return 2.5 * op["shape"][0] * op["shape"][1]


def _planless_check(op, data, y):
    if op["op"] in ("conv_fft", "conv_os") and not op.get("big"):
        want = ck.int_conv(data[0], data[1]).astype(np.float64)
        osk.check_exact(y.ravel(order="F"), want.ravel(order="F"), False, what=op["id"])
    if op["op"] == "per2" and op["ptype"]:
        S, E = ck.per2_ref(data[0].astype(np.float64), op["nfft"][0], op["nfft"][1], F32)
        tot, bnd, pop, kmax = ck.radial_ref(S, E, op["nfft"][0], op["nfft"][1], _per2_r(op), F32)
        ref = tot / pop if op["ptype"] == 2 else tot
        bd = bnd / pop if op["ptype"] == 2 else bnd
        assert y.size == kmax and bool(np.all(np.abs(y.astype(np.float64) - ref) <= bd)), op["id"]


@pytest.mark.gpu
def test_planless_cache_arena_and_budget(dsp):
    """The plan-less calls through more cuFFT keys than the cache holds, the arena grown, shrunk and regrown, the N-D
    overlap-save budget changed: a revisited call equals its first run bit for bit (radial periodograms: the bound)."""
    from dspb200 import device
    seq = planless_sequence()
    model = lru_model(seq)
    first = {}
    revisited_after_eviction = 0
    evicted = set()
    try:
        for i, op in enumerate(seq):
            evicted |= set(model[i]["evicted"])
            if op["op"] == "set_budget":
                dsp._lib.conv_nd_os_set_budget(op["budget"])
                continue
            if op["op"] == "refuse":
                u = np.ones((10, 10), F32)
                b = Bufs()
                gu, go = b.inp(F32, u, _rng("refuse")), b.out(F32, 12 * 12)
                refused(dsp, lambda: dsp._lib.conv_nd_dev(F32, (10, 10), gu.ptr, (3, 3), gu.ptr, (2, 2), go.ptr, True, 0))
                continue
            data = _planless_data(op)
            y = _planless_run(dsp, op, data, _rng("pl-guard", i))
            if op["id"] not in first:
                _planless_check(op, data, y)
                first[op["id"]] = y
                continue
            if op["op"] == "per2" and op["ptype"]:
                _planless_check(op, data, y)
            else:
                assert same_bits(y, first[op["id"]]), (i, op["id"])
            if set(planless_keys(op)) & evicted:
                revisited_after_eviction += 1
            evicted -= set(planless_keys(op))
        assert revisited_after_eviction >= 4, revisited_after_eviction
    finally:
        dsp._lib.conv_nd_os_set_budget(DEFAULT_BUDGET)
        device.empty_cache()
