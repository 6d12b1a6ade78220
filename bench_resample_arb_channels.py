"""Arbitrary-rate resampling of many channels in one launch against a per-channel loop, on one GPU.

For each shape, the len x nchan matrix is generated on the device from a seed and resampled per column two ways:
  * batched: one resample(D, rate, h, dims=0) call on the device matrix (dspb200_resample_arb_batch_exec_dev);
  * loop:    one resample(column, rate, h) call per device column (dspb200_resample_arb_exec_dev).
Both are timed end to end with CUDA events (each public call builds its plan and ends with a synchronise), after warm-up,
alternating the two forms.  A second pair of numbers, "launch only", times the device work alone with one plan: one batched
launch into a device buffer against the per-column launches, without synchronisation in between.  The batched outputs
are compared with the loop's bit for bit in the same run.

The last shape is a single vector timed through the single-vector entry only (plan.exec_dev), which older builds of the
library also have, so the same script can time them.  It reports launch-only numbers.

The reported rate is algorithmic: (input bytes + output bytes) / launch-only time, and its fraction of 3.35 TB/s.
Prints one JSON line per shape with the card name, power limit and max SM clock.  Writes nothing unless --out is given.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_TBS = 3.35            # H100 SXM HBM3, data sheet

# (nchan, len, dtype, rate, taps dtype: "float32" = resample_filter(rate, 32) in Float32, "default" = its Float64 taps).
# 1024 x 2^14: short channels, where the loop is bound by launches; 1/55.55: both tap banks (1 MB) in global memory.
SHAPES = {
    "multi": [
        (64, 1 << 20, "float32", 0.9802414928649835, "float32"),
        (1024, 1 << 14, "float32", 1.2957, "float32"),
        (8, 1 << 23, "complex64", 2.618, "float32"),
        (16, 1 << 20, "float32", 1 / 55.55, "default"),
    ],
    "single": [
        (1, 1 << 26, "complex64", 0.7312, "float32"),
    ],
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:      # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def call_args(dsp, h, rate, nx):
    """(outLen, samples read per column, n0, acc0, delta) of resample(x, rate, h) on a column of nx samples: a fresh
    FIRFilter after undelay!, the column zero-padded to inputlength(outLen, RoundUp) + 1 samples."""
    sf = dsp.FIRFilter(h, rate, 32)
    outlen = math.ceil(nx * rate)
    sf.setphase(sf.timedelay())
    npad = max(sf.inputlength(outlen, round_up=True), 0) + 1
    return outlen, min(nx, npad), sf.input_deficit - 1, sf.phi_accumulator, sf.delta


def timed(torch, fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    res = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), res


def stats(t, nbytes):
    out = {}
    for key, v in t.items():
        ms = float(np.median(v))
        out[key] = {"ms": round(ms, 4), "ms_min": round(float(np.min(v)), 4)}
        if key.endswith("launch"):
            out[key].update({"tb_per_s": round(nbytes / ms / 1e9, 3), "share_of_3.35_tb_per_s": round(nbytes / ms / 1e9 / PEAK_TBS, 3)})
    return out


def run_shape(torch, dsp, nchan, length, dtname, rate, taps, reps, warmup):
    dt = np.dtype(dtname)
    h = dsp.resample_filter(rate, 32)
    if taps == "float32":
        h = h.astype(np.float32)
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    if dt.kind == "c":
        x = torch.view_as_complex(torch.randn(nchan, length, 2, device="cuda", generator=g, dtype=torch.float32))
    else:
        x = torch.randn(nchan, length, device="cuda", generator=g, dtype=torch.float32)
    # (nchan, len) row-major = column-major len x nchan: column c starts c * len samples in
    D = dsp.DeviceArray((length, nchan), dt, _base=x, _ptr=x.data_ptr())
    cols = [dsp.DeviceArray((length,), dt, _base=x, _ptr=x.data_ptr() + c * length * dt.itemsize) for c in range(nchan)]
    outlen, m, n0, acc0, delta = call_args(dsp, h, rate, length)
    plan = dsp._lib.ResampleArbPlan(dt, h, 32)
    odt = np.dtype(plan.out_dtype)
    dout = dsp.DeviceArray((outlen, nchan), odt)
    nbytes = nchan * (length * dt.itemsize + outlen * odt.itemsize)

    def loop_launch():
        for c in range(nchan):
            plan.exec_dev(cols[c].ptr, m, n0, acc0, delta, dout.ptr + c * outlen * odt.itemsize, outlen, 0)

    res = {"shape": f"{nchan} x {length} {dtname}", "rate": rate, "taps": f"{h.size} {h.dtype}",
           "taps_per_phase": -(-h.size // 32)}
    t = {"loop_launch": []}
    if nchan == 1:
        for _ in range(warmup):
            loop_launch()
        for _ in range(reps):
            t["loop_launch"].append(timed(torch, loop_launch)[0])
        res.update(stats(t, nbytes))
        res["single_vector_launch"] = res.pop("loop_launch")
        return res

    def batched():
        return dsp.resample(D, rate, h, dims=0)

    def loop():
        return [dsp.resample(cols[c], rate, h) for c in range(nchan)]

    def batched_launch():
        plan.exec_batch_dev(D.ptr, m, length, nchan, n0, acc0, delta, dout.ptr, outlen, 0)

    for _ in range(warmup):
        batched(); loop(); batched_launch(); loop_launch()
    t = {"batched": [], "loop": [], "batched_launch": [], "loop_launch": []}
    yb = yl = None
    for _ in range(reps):
        ms, yb = timed(torch, batched); t["batched"].append(ms)
        ms, yl = timed(torch, loop); t["loop"].append(ms)
        ms, _ = timed(torch, batched_launch); t["batched_launch"].append(ms)
        ms, _ = timed(torch, loop_launch); t["loop_launch"].append(ms)
    hb = yb.to_host()
    res["bit_equal_batched_vs_loop"] = bool(all(np.array_equal(hb[:, c], yl[c].to_host()) for c in range(nchan)))
    res.update(stats(t, nbytes))
    res["speedup_end_to_end"] = round(res["loop"]["ms"] / res["batched"]["ms"], 2)
    res["speedup_launch_only"] = round(res["loop_launch"]["ms"] / res["batched_launch"]["ms"], 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", choices=["all", "multi", "single"], default="all")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_resample_arb_channels.py needs a CUDA device")
    gpu = card()
    shapes = SHAPES["multi"] + SHAPES["single"] if args.shapes == "all" else SHAPES[args.shapes]
    lines = []
    for shape in shapes:
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
