"""filtfilt and alignsignals of device-resident channel matrices against the host calls, on one GPU.

  * filtfilt of a 2^20 x 64 Float32 matrix with a 33-tap filter (65 taps of conv(b, reverse(b)): the time-domain FIR
    kernel) and a 257-tap filter (513 taps: overlap-save).  Device: one filtfilt call on the DeviceArray (extension, filter
    and crop in HBM).  Host: filtfilt of the same matrix from host memory (numpy extension, copies over PCIe, the same
    GPU filter).
  * alignsignals of 64 channels of 2^20 Float32 samples against one 4096-sample reference.  Device: one alignsignals call
    on the DeviceArray (one correlation launch for every channel, one peak-search launch, one shift launch, one
    synchronisation for the delays).  Host: a loop of 64 alignsignals calls on host vectors.

Each form is timed with CUDA events around the whole call, after warm-up, and reported as the median (and minimum) over
--reps runs.  Every line checks the device result against the host call in the same run: filtfilt bit for bit, alignsignals
delays and aligned channels exactly (each channel holds the reference at a known delay above the noise, so the peak is
unambiguous).  Prints one JSON line per workload with the card name and power limit read in the same run.  Writes nothing.
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

LEN, NCHAN, NREF = 1 << 20, 64, 4096


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:      # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def timer(torch, reps, warmup):
    def run(fn):
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
        return {"ms": round(float(np.median(ts)), 3), "ms_min": round(float(np.min(ts)), 3), "reps": reps}, res
    return run


def bench_filtfilt(torch, dsp, nb, reps, host_reps, warmup):
    rng = np.random.default_rng(nb)
    b = (rng.standard_normal(nb) / nb).astype(np.float32)
    x = rng.standard_normal((LEN, NCHAN)).astype(np.float32, order="F")
    dx = dsp.to_device(x)
    dev_t, dev_y = timer(torch, reps, warmup)(lambda: dsp.filtfilt(b, dx))
    host_t, host_y = timer(torch, host_reps, 1)(lambda: dsp.filtfilt(b, x))
    got = dev_y.to_host()
    ntaps = 2 * nb - 1
    return {"workload": f"filtfilt {LEN} x {NCHAN} float32, {nb} taps ({ntaps} taps of conv(b, reverse(b)))",
            "route": "overlap-save" if ntaps > dsp.SMALL_FILT_CUTOFF else "time-domain FIR",
            "device": dev_t, "host": host_t, "speedup": round(host_t["ms"] / dev_t["ms"], 2),
            "check_bit_identical_to_host": bool(np.array_equal(got.view(np.uint32), host_y.view(np.uint32)))}


def bench_alignsignals(torch, dsp, reps, host_reps, warmup):
    rng = np.random.default_rng(5)
    y = rng.standard_normal(NREF).astype(np.float32)
    x = (0.1 * rng.standard_normal((LEN, NCHAN))).astype(np.float32, order="F")
    true = rng.integers(0, LEN - NREF, NCHAN)
    for c, s in enumerate(true):
        x[s:s + NREF, c] += y
    dx = dsp.to_device(x)

    def host_loop():
        out = np.empty_like(x)
        d = np.empty(NCHAN, dtype=np.int64)
        for c in range(NCHAN):
            out[:, c], d[c] = dsp.alignsignals(x[:, c], y)
        return out, d

    dev_t, (dev_a, dev_d) = timer(torch, reps, warmup)(lambda: dsp.alignsignals(dx, y))
    host_t, (host_a, host_d) = timer(torch, host_reps, 1)(host_loop)
    return {"workload": f"alignsignals {LEN} x {NCHAN} float32 against a {NREF}-sample reference",
            "route": dsp.clients._xcorr_route(LEN, NREF), "device": dev_t, "host_loop_of_64_calls": host_t,
            "speedup": round(host_t["ms"] / dev_t["ms"], 2),
            "check_delays_equal_host": bool(np.array_equal(dev_d, host_d) and np.array_equal(dev_d, true)),
            "check_aligned_equal_host": bool(np.array_equal(dev_a.to_host(), host_a))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_clients.py needs a CUDA device")
    gpu = card()
    ok = True
    for res in (bench_filtfilt(torch, dsp, 33, args.reps, args.host_reps, args.warmup),
                bench_filtfilt(torch, dsp, 257, args.reps, args.host_reps, args.warmup),
                bench_alignsignals(torch, dsp, args.reps, args.host_reps, args.warmup)):
        res["gpu"] = gpu
        ok &= all(v for k, v in res.items() if k.startswith("check_"))
        print(json.dumps(res), flush=True)
    if not ok:
        raise SystemExit("a device result differs from the host call")


if __name__ == "__main__":
    main()
