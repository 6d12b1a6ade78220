"""Batched Welch over channels against a per-channel loop, on one GPU.

For each shape, the len x nchan matrix is generated on the device and Welch-averaged per column two ways:
  * batched: one welch_pgram call on the device matrix (dspb200_welch_batch_exec_dev), power copied to the host;
  * loop:    one welch_pgram call per column (dspb200_welch_exec_dev) that reuses one WelchConfig, power copied each time.
Both are timed end to end with CUDA events (each call ends with its device-to-host copy and a synchronise), after warm-up,
alternating the two forms.  A second pair of numbers, "launch only", times the device work alone: one batched launch
sequence into a device buffer against the per-column launch sequences, without copies or synchronisation in between.
The batched power is checked against the loop's in the same run (norm-relative, per column).

Prints one JSON line per shape with the card name and power limit.  Writes nothing unless --out is given.
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

PEAK_TBS = 3.35            # H100 SXM HBM3, data sheet

# (nchan, len, dtype, n, noverlap, onesided)
SHAPES = [
    (64, 1 << 22, "float32", 4096, 2048, True),
    (1024, 1 << 16, "float32", 1024, 512, True),
    (8, 1 << 24, "complex64", 4096, 2048, False),
]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:      # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def run_shape(torch, dsp, nchan, length, dtname, n, nov, onesided, reps, warmup):
    dt = np.dtype(dtname)
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    if dt.kind == "c":
        x = torch.view_as_complex(torch.randn(nchan, length, 2, device="cuda", generator=g, dtype=torch.float32))
    else:
        x = torch.randn(nchan, length, device="cuda", generator=g, dtype=torch.float32)
    # (nchan, len) row-major = column-major len x nchan: column c starts c * len samples in
    D = dsp.DeviceArray((length, nchan), dt, _base=x, _ptr=x.data_ptr())
    cols = [dsp.DeviceArray((length,), dt, _base=x, _ptr=x.data_ptr() + c * length * dt.itemsize) for c in range(nchan)]
    cfg = dsp.WelchConfig(length, dt, n=n, noverlap=nov, onesided=onesided, window=dsp.hanning)
    nout = cfg.freq.size
    k = dsp.arraysplit_count(length, n, nov)
    r = k * cfg.r
    odt = dsp.fftabs2type(dt)
    dout = dsp.DeviceArray((nout, nchan), odt)

    def batched():
        return dsp.welch_pgram(D, cfg).power

    def loop():
        out = np.empty((nout, nchan), dtype=odt, order="F")
        for c in range(nchan):
            out[:, c] = dsp.welch_pgram(cols[c], cfg).power
        return out

    def batched_launch():
        cfg.plan.welch_batch_dev(D.ptr, length, nchan, r, dout.ptr, 0)

    def loop_launch():
        for c in range(nchan):
            cfg.plan.welch_dev(cols[c].ptr, length, r, dout.ptr + c * nout * odt.itemsize, 0)

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        res = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), res

    for _ in range(warmup):
        batched(); loop(); batched_launch(); loop_launch()
    torch.cuda.synchronize()
    t = {"batched": [], "loop": [], "batched_launch": [], "loop_launch": []}
    pb = pl = None
    for _ in range(reps):
        ms, pb = timed(batched); t["batched"].append(ms)
        ms, pl = timed(loop); t["loop"].append(ms)
        ms, _ = timed(batched_launch); t["batched_launch"].append(ms)
        ms, _ = timed(loop_launch); t["loop_launch"].append(ms)
    err = 0.0
    for c in range(nchan):
        d = np.linalg.norm(pb[:, c].astype(np.float64) - pl[:, c])
        m = max(np.linalg.norm(pb[:, c].astype(np.float64)), np.linalg.norm(pl[:, c].astype(np.float64)))
        err = max(err, d / m if m > 0 else d)
    samples = nchan * length
    nbytes = samples * dt.itemsize
    res = {"shape": f"{nchan} x {length} {dtname}", "n": n, "noverlap": nov, "window": "hanning", "segments_per_channel": k,
           "max_column_relerr_batched_vs_loop": err, "bit_equal_batched_vs_loop": bool(np.array_equal(pb, pl))}
    for key, v in t.items():
        ms = float(np.median(v))
        res[key] = {"ms": round(ms, 4), "ms_min": round(float(np.min(v)), 4), "gsamples_per_s": round(samples / ms / 1e6, 2),
                    "tb_per_s": round(nbytes / ms / 1e9, 3), "share_of_3.35_tb_per_s": round(nbytes / ms / 1e9 / PEAK_TBS, 3)}
    res["speedup_end_to_end"] = round(res["loop"]["ms"] / res["batched"]["ms"], 2)
    res["speedup_launch_only"] = round(res["loop_launch"]["ms"] / res["batched_launch"]["ms"], 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_welch_channels.py needs a CUDA device")
    gpu = card()
    lines = []
    for shape in SHAPES:
        res = run_shape(torch, dsp, *shape, reps=args.reps, warmup=args.warmup)
        res["gpu"] = gpu
        lines.append(json.dumps(res))
        print(lines[-1], flush=True)
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
