"""Streaming FIR through a device-resident DF2TFilter against one stateless filt over the whole signal, on one GPU.

Workload: a 64-channel Float32 signal of 2^20 samples per channel in device memory, the 257-tap C1 filter.  It is filtered
  * one-shot:  filt(b, 1, X) over the whole 2^20 x 64 column-major matrix (one stateless launch);
  * streamed:  a device DF2TFilter fed consecutive blocks of C samples x 64 channels (C = 4096 and 65536), each block a
               column-major C x 64 array as an acquisition would deliver it; one stateful launch per block.
Each block computes C + 256 outputs per channel (the last 256 are the carried state), so the expected extra work is
(nb - 1) / C of the one-shot outputs plus one launch per block.  Times are CUDA events around each form (device-resident
inputs, preallocated outputs, no copies), after warm-up, the forms alternating: the one-shot time is its launch; the
streamed time is the sequence of Python `filt_` calls, so it includes the front end's host-side work for every block as
well as the launches.  In the same run the streamed outputs are copied back and compared with the one-shot output for
bit equality.

Prints one JSON line per block size with the card name and power limit.  Writes nothing unless --out is given.
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


def c1_taps():
    n = np.arange(257) - 128
    return (0.5 * np.sinc(0.5 * n) * np.hamming(257)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=64)
    ap.add_argument("--log2n", type=int, default=20)
    ap.add_argument("--chunks", default="4096,65536")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_fir_stream.py needs a CUDA device")
    gpu = card()
    nch, n = args.channels, 1 << args.log2n
    b = c1_taps()
    nb = b.size
    x = np.random.default_rng(2024).standard_normal((n, nch)).astype(np.float32)
    X = dsp.to_device(x)
    Y = dsp.DeviceArray((n, nch), np.float32)
    plan = dsp._lib.FirPlan(b)
    pr = dsp.PolynomialRatio(b, np.float32(1))

    def one_shot():
        plan.exec_dev(X.ptr, n, nch, Y.ptr, 0)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    lines = []
    for c in (int(v) for v in args.chunks.split(",")):
        if n % c:
            raise SystemExit(f"block length {c} must divide {n}")
        nblk = n // c
        # blocks laid out one after the other, each a column-major c x nch array
        xb = np.concatenate([np.asfortranarray(x[k * c:(k + 1) * c]).ravel(order="F") for k in range(nblk)])
        XB = dsp.to_device(xb)
        YB = dsp.DeviceArray(xb.shape, np.float32)
        step = c * nch * 4
        xin = [dsp.DeviceArray((c, nch), np.float32, _base=XB, _ptr=XB.ptr + k * step) for k in range(nblk)]
        yout = [dsp.DeviceArray((c, nch), np.float32, _base=YB, _ptr=YB.ptr + k * step) for k in range(nblk)]
        f = dsp.DF2TFilter(pr, (nch,), device=True)

        def streamed():
            for k in range(nblk):
                dsp.filt_(yout[k], f, xin[k])

        for _ in range(args.warmup):
            one_shot(); streamed()
        t = {"one_shot": [], "streamed": []}
        for _ in range(args.reps):
            t["one_shot"].append(timed(one_shot))
            t["streamed"].append(timed(streamed))
        # bit equality: a fresh filter over the whole stream against the one-shot output
        f = dsp.DF2TFilter(pr, (nch,), device=True)
        l0 = dsp.launch_count()
        streamed()
        launches = dsp.launch_count() - l0
        one_shot()
        yb = YB.to_host().reshape(nblk, nch, c)                 # block k, channel j, sample i
        ys = np.ascontiguousarray(yb.transpose(0, 2, 1)).reshape(n, nch)
        y1 = Y.to_host()
        res = {"workload": f"{nch} ch x 2^{args.log2n} Float32, {nb} taps, device DF2TFilter in blocks of {c}",
               "blocks": nblk, "launches_per_stream": launches, "bit_equal_streamed_vs_one_shot": bool(np.array_equal(ys, y1)),
               "extra_outputs_fraction": round((nb - 1) / c, 5)}
        for key, v in t.items():
            ms = float(np.median(v))
            res[key] = {"ms": round(ms, 4), "ms_min": round(float(np.min(v)), 4), "gsamples_per_s": round(n * nch / ms / 1e6, 2)}
        res["streamed_over_one_shot"] = round(res["streamed"]["ms"] / res["one_shot"]["ms"], 3)
        res["gpu"] = gpu
        lines.append(json.dumps(res))
        print(lines[-1], flush=True)
        del XB, YB, xin, yout
    plan.close()
    if args.out:
        with open(args.out, "w") as fo:
            fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
