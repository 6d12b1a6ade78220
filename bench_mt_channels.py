"""Multitaper estimates of channel matrices against per-channel and per-taper calls, on one GPU.

Lines (each one checks its outputs in the same run):
  * mt_spectrogram, 64 x 2^22 Float32 (n = nfft = 1024, 75 % overlap, nw = 4: 7 tapers), device matrix in and out:
      - batched: one mt_spectrogram call on the matrix (one launch);
      - per taper: the same sum from public calls -- one batched spectrogram(S; window = w_t / sqrt(r_t), fs = 1 / norm2_t,
        so that its r is 1) per taper, added in taper order on the host (the adds are not timed); must be bit-identical;
      - loop: one vector mt_spectrogram call per channel; every column must be bit-identical to the matrix call's.
  * mt_pgram, 1024 channels x 2048 Float32 (fused) and 64 channels x 2^16 Float32 (cuFFT), against a loop of vector calls
    that reuses one MTConfig; fused columns must be bit-identical, cuFFT columns within 1e-6 (norm-relative) and the
    bit-equality is reported.
Times are CUDA-event milliseconds of the whole call (median of --reps, after --warmup), which for these device-resident
calls includes plan creation and the call's final synchronise.  Prints one JSON line per workload with the card name and
power limit.  Writes nothing unless --out is given.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:      # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def device_matrix(torch, dsp, nchan, length, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    x = torch.randn(nchan, length, device="cuda", generator=g, dtype=torch.float32)
    # (nchan, len) row-major = column-major len x nchan: column c starts c * len samples in
    D = dsp.DeviceArray((length, nchan), np.float32, _base=x, _ptr=x.data_ptr())
    cols = [dsp.DeviceArray((length,), np.float32, _base=x, _ptr=x.data_ptr() + c * length * 4) for c in range(nchan)]
    return D, cols


def timed(torch, fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts, res = [], None
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        res = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return {"ms": round(float(np.median(ts)), 3), "ms_min": round(float(np.min(ts)), 3)}, res


def bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def spectrogram_line(torch, dsp, reps, warmup):
    nchan, length, n, nov, nw = 64, 1 << 22, 1024, 768, 4
    D, cols = device_matrix(torch, dsp, nchan, length, 4)
    cfg = dsp.MTConfig(np.float32, n, nw=nw, noverlap=nov)
    nt = cfg.ntapers
    k = dsp.arraysplit_count(length, n, nov)
    t_mt, P = timed(torch, lambda: dsp.mt_spectrogram(D, n, nov, nw=nw).power, reps, warmup)
    Ph = P.to_host()
    del P
    rows = [cfg.window[:, t] / np.sqrt(cfg.r[t]) for t in range(nt)]
    fss = [1.0 / float(np.sum(w * w)) for w in rows]          # r = fs * norm2 = 1 (to Float32 rounding of 1/r and 2/r)
    assert all(np.float32(1.0 / (fs * np.sum(w * w))) == 1 and np.float32(2.0 / (fs * np.sum(w * w))) == 2 for fs, w in zip(fss, rows))

    def per_taper():
        return [dsp.spectrogram(D, n, nov, window=w, fs=fs).power for w, fs in zip(rows, fss)]
    t_taper, outs = timed(torch, per_taper, reps, warmup)
    acc = None
    for o in outs:
        h = o.to_host()
        acc = h if acc is None else acc + h                   # Float32 adds, taper order
    del outs
    taper_equal = bits_equal(acc, Ph)
    del acc

    def loop():
        return [dsp.mt_spectrogram(cols[c], n, nov, nw=nw).power for c in range(nchan)]
    t_loop, outs = timed(torch, loop, max(1, reps // 2), 1)
    loop_equal = all(bits_equal(outs[c].to_host(), Ph[:, :, c]) for c in range(nchan))
    del outs
    assert taper_equal and loop_equal, (taper_equal, loop_equal)
    in_b, out_b = nchan * length * 4, nchan * k * cfg.freq.size * 4
    return {"workload": f"mt_spectrogram {nchan} x 2^22 float32, n = nfft = {n}, noverlap {nov}, nw {nw} ({nt} tapers)",
            "segments_per_channel": k, "batched": t_mt, "per_taper_public_calls": t_taper, "loop_vector_calls": t_loop,
            "bit_equal_per_taper_sum": taper_equal, "bit_equal_loop": loop_equal,
            "hbm_bytes_one_pass": in_b + out_b, "tb_per_s_one_pass": round((in_b + out_b) / t_mt["ms"] / 1e9, 3),
            "speedup_vs_per_taper": round(t_taper["ms"] / t_mt["ms"], 2), "speedup_vs_loop": round(t_loop["ms"] / t_mt["ms"], 2)}


def pgram_line(torch, dsp, nchan, length, reps, warmup):
    D, cols = device_matrix(torch, dsp, nchan, length, 5)
    cfg = dsp.MTConfig(np.float32, length, nw=4, nfft=dsp.nextfastfft(length))
    t_mt, P = timed(torch, lambda: dsp.mt_pgram(D, cfg).power.to_host(), reps, warmup)

    def loop():
        out = np.empty(P.shape, dtype=np.float32, order="F")
        for c in range(nchan):
            out[:, c] = dsp.mt_pgram(cols[c], cfg).power.to_host()
        return out
    t_loop, L = timed(torch, loop, max(1, reps // 2), 1)
    err = max(float(np.linalg.norm(P[:, c].astype(np.float64) - L[:, c]) / np.linalg.norm(L[:, c].astype(np.float64)))
              for c in range(nchan))
    equal = bits_equal(P, L)
    fused = cfg.plan.fused
    assert (equal if fused else err < 1e-6), (equal, err)
    return {"workload": f"mt_pgram {nchan} x {length} float32, nfft {cfg.nfft} ({'fused' if fused else 'cuFFT'}), "
                        f"nw 4 ({cfg.ntapers} tapers)",
            "batched": t_mt, "loop_vector_calls": t_loop, "bit_equal_loop": equal, "max_column_relerr_vs_loop": err,
            "speedup_vs_loop": round(t_loop["ms"] / t_mt["ms"], 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_mt_channels.py needs a CUDA device")
    gpu = card()
    lines = []
    for fn in (lambda: spectrogram_line(torch, dsp, args.reps, args.warmup),
               lambda: pgram_line(torch, dsp, 1024, 2048, args.reps, args.warmup),
               lambda: pgram_line(torch, dsp, 64, 1 << 16, args.reps, args.warmup)):
        res = fn()
        res["gpu"] = gpu
        lines.append(json.dumps(res))
        print(lines[-1], flush=True)
        dsp.device.empty_cache()
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
