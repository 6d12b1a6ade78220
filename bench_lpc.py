"""lpc / arburg on device-resident channel matrices, on one GPU.

Workloads (all device-resident, CUDA events after warm-up, the median of alternating rounds):
  * frames:   65 536 frames x 512 samples, Float32 and Float64, p = 16, Burg (the shared-memory path) and Levinson;
  * long:     64 channels x 2^20 samples, Float32, p = 32, Burg (the streamed path, a cluster of 8 CTAs per column);
  * matrix vs loop: one matrix call over 256 columns of 512 samples against 256 vector calls, outputs checked bit for bit
    in the run.
Reported: ms per call, Gsamples/s, and the share of the larger of two bounds (bounds()): the HBM bound, the input read once
and the outputs written once at the data sheet's 3.35 TB/s; the compute bound, 6 p flops per real sample for Burg (the error
update and the fused dot of each order: three fmas) and 2 (p + 1) per real sample for the autocorrelation of Levinson,
against the data-sheet FP32 (67 TFLOP/s) and FP64 (34 TFLOP/s) rates of the H100 SXM.  A complex sample counts as four real
ones for flops.  Prints one JSON line per workload with the card name and power limit.  Writes nothing unless --out is given.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_fir_stream import card  # noqa: E402

HBM = 3.35e12
PEAK = {"float32": 67e12, "float64": 34e12}


def bounds(dtype, n, ncols, p, method):
    """(HBM-bound seconds, compute-bound seconds) of one call."""
    dt = np.dtype(dtype)
    esz = dt.itemsize
    rsz = 4 if dt in (np.float32, np.complex64) else 8
    na = p + 1 if method == "burg" else p
    nbytes = n * ncols * esz + na * ncols * esz + ncols * rsz
    real_samples = n * ncols * (4 if dt.kind == "c" else 1)
    flops = (6 * p if method == "burg" else 2 * (p + 1)) * real_samples
    peak = PEAK["float32" if rsz == 4 else "float64"]
    return nbytes / HBM, flops / peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_lpc.py needs a CUDA device")
    gpu = card()

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def rounds(fns):
        """median ms of each fn over args.reps alternating rounds, after args.warmup untimed ones"""
        for _ in range(args.warmup):
            for f in fns:
                f()
        torch.cuda.synchronize()
        ts = [[] for _ in fns]
        for _ in range(args.reps):
            for i, f in enumerate(fns):
                ts[i].append(timed(f))
        return [statistics.median(t) for t in ts]

    rng = np.random.default_rng(0)
    lines = []

    def emit(res):
        line = json.dumps(res)
        print(line, flush=True)
        lines.append(line)

    def workload(name, dtype, n, ncols, p, methods):
        x = dsp.to_device(np.asfortranarray(rng.standard_normal((n, ncols)).astype(dtype)))
        fns = [(lambda m=m: dsp.lpc(x, p, dsp.LPCBurg() if m == "burg" else dsp.LPCLevinson())) for m in methods]
        ms = rounds(fns)
        for m, t in zip(methods, ms):
            hb, cb = bounds(dtype, n, ncols, p, m)
            bound, which = (hb, "hbm") if hb >= cb else (cb, "compute")
            emit({"workload": name, "dtype": np.dtype(dtype).name, "method": m, "n": n, "ncols": ncols, "p": p, "ms": round(t, 4),
                  "gsamples_per_s": round(n * ncols / (t * 1e-3) / 1e9, 3), "bound_ms": round(bound * 1e3, 4), "bound": which,
                  "share_of_bound": round(bound * 1e3 / t, 4), "card": gpu})

    for dt in (np.float32, np.float64):
        workload("frames", dt, 512, 65536, 16, ("burg", "levinson"))
    workload("long", np.float32, 1 << 20, 64, 32, ("burg",))

    # one matrix call against a loop of vector calls, bit for bit
    n, ncols, p = 512, 256, 16
    xh = np.asfortranarray(rng.standard_normal((n, ncols)).astype(np.float32))
    x = dsp.to_device(xh)
    cols = [dsp.to_device(xh[:, c].copy()) for c in range(ncols)]
    res = {}

    def matrix():
        res["m"] = dsp.lpc(x, p)

    def loop():
        res["l"] = [dsp.lpc(c, p) for c in cols]

    tm, tl = rounds([matrix, loop])
    am, em = res["m"][0].to_host(), res["m"][1].to_host()
    same = all(np.array_equal(am[:, c].view(np.int32), a.to_host().view(np.int32)) and
               np.array_equal(em[c:c + 1].view(np.int32), np.atleast_1d(e.to_host()).view(np.int32))
               for c, (a, e) in enumerate(res["l"]))
    emit({"workload": "matrix_vs_loop", "dtype": "float32", "method": "burg", "n": n, "ncols": ncols, "p": p,
          "matrix_ms": round(tm, 4), "loop_ms": round(tl, 4), "speedup": round(tl / tm, 2), "bit_identical": bool(same), "card": gpu})
    if not same:
        raise SystemExit("matrix and vector calls differ")
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
