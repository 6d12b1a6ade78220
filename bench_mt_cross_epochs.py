"""Multitaper cross spectra of many epochs in one call against a loop of matrix calls, on one GPU.

Workload: a device-resident n_channels x n_samples x n_epochs array (64 x 1024 x 512 by default), Float32 and Float64, dpss
tapers with nw = 4 (7 tapers), nfft = n_samples, demean on, over the full frequency range and over a narrow freq_range.
Forms timed, each with CUDA events after warm-up, the median of alternating rounds:
  * epochs: one dspb200_mt_cross_spectra_epochs call (the epoch mean);
  * loop:   one dspb200_mt_cross_spectra_exec_dev matrix call per epoch, each added to a running device sum (torch adds in
            epoch order), then the real and imaginary parts divided by n_epochs -- what a caller without the epoch call
            writes.  Its result is checked bit for bit against the epoch call in the same run;
  * matrix: the matrix call at 256 channels x 4096 samples (one epoch);
  * acc:    the accumulate kernel (cs_acc_kernel) alone, its device time summed from a torch.profiler trace of epoch calls
            (the kernel has no entry point of its own).
FLOP/s counts 8 n_channels^2 nf ntapers n_epochs (one complex multiply-add per taper, epoch and output), set against the
data-sheet FP32 (67 TFLOP/s) and FP64 (34 TFLOP/s) rates of the H100 SXM.  Prints one JSON line per (eltype, range) with
the card name and power limit.  Writes nothing unless --out is given.
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

PEAK = {"float32": 67e12, "float64": 34e12}        # H100 SXM data sheet, non-tensor


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nchan", type=int, default=64)
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--epochs", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dtypes", default="float32,float64")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_mt_cross_epochs.py needs a CUDA device")
    gpu = card()
    nchan, n, E = args.nchan, args.n, args.epochs

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    lines = []
    for dname in args.dtypes.split(","):
        dt = np.dtype(dname)
        tdt = torch.float32 if dt == np.float32 else torch.float64
        cdt = torch.complex64 if dt == np.float32 else torch.complex128
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn(nchan * n * E, generator=g, device="cuda", dtype=tdt) + 0.5      # channel fastest, then sample, epoch
        mt = dsp.MTConfig(dt, n, nfft=n, nw=4)
        big = dsp.MTConfig(dt, 4096, nfft=4096, nw=4)
        xb = torch.randn(256 * 4096, generator=g, device="cuda", dtype=tdt)
        for rname, frange in (("full", None), ("narrow", (0.10, 0.15))):
            cfg = dsp.MTCrossSpectraConfig(nchan, mt, demean=True, freq_range=frange)
            f_lo, nf, K = cfg.freq_lo, cfg.nfreq, mt.ntapers
            out = torch.empty((nf, nchan, nchan), dtype=cdt, device="cuda")
            m = torch.empty_like(out)
            acc = torch.empty_like(out)
            ref = torch.empty_like(out)
            step = nchan * n * x.element_size()

            def epochs():
                mt.plan.cross_spectra_epochs_dev(x.data_ptr(), nchan, E, True, f_lo, nf, False, out.data_ptr())

            def loop():
                for e in range(E):
                    mt.plan.cross_spectra_dev(x.data_ptr() + e * step, nchan, True, f_lo, nf, False, m.data_ptr())
                    if e == 0:
                        acc.copy_(m)
                    else:
                        acc.add_(m)
                torch.view_as_real(ref).copy_(torch.view_as_real(acc) / E)

            cfgb = dsp.MTCrossSpectraConfig(256, big, demean=True, freq_range=frange)
            outb = torch.empty((cfgb.nfreq, 256, 256), dtype=cdt, device="cuda")

            def matrix():
                big.plan.cross_spectra_dev(xb.data_ptr(), 256, True, cfgb.freq_lo, cfgb.nfreq, False, outb.data_ptr())

            forms = {"epochs": epochs, "loop": loop, "matrix": matrix}
            for _ in range(args.warmup):
                for fn in forms.values():
                    fn()
            torch.cuda.synchronize()
            same = bool(torch.equal(torch.view_as_real(out), torch.view_as_real(ref)))
            times = {k: [] for k in forms}
            for _ in range(args.reps):
                for k, fn in forms.items():
                    times[k].append(timed(fn))
            med = {k: statistics.median(v) for k, v in times.items()}
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    epochs()
                torch.cuda.synchronize()
            acc_us = sum(ev.device_time_total for ev in prof.key_averages() if "cs_acc_kernel" in ev.key) / args.reps
            flop = 8.0 * nchan * nchan * nf * K * E
            flopb = 8.0 * 256 * 256 * cfgb.nfreq * big.ntapers
            res = {"dtype": dname, "range": rname, "nchan": nchan, "n": n, "epochs": E, "ntapers": K, "nf": nf,
                   "epochs_ms": round(med["epochs"], 3), "loop_ms": round(med["loop"], 3),
                   "speedup": round(med["loop"] / med["epochs"], 2), "bitwise_equal": same,
                   "epochs_tflops": round(flop / med["epochs"] * 1e-9, 3),
                   "acc_kernel_ms": round(acc_us * 1e-3, 3), "acc_kernel_tflops": round(flop / acc_us * 1e-6, 3) if acc_us else None,
                   "acc_share_of_peak": round(flop / acc_us * 1e6 / PEAK[dname], 3) if acc_us else None,
                   "matrix_256x4096_ms": round(med["matrix"], 3), "matrix_256x4096_tflops": round(flopb / med["matrix"] * 1e-9, 3),
                   "gpu": gpu}
            line = json.dumps(res)
            print(line, flush=True)
            lines.append(line)
            if not same:
                raise SystemExit("the epoch call and the loop of matrix calls differ")
        del x, xb
        torch.cuda.empty_cache()
        dsp.device.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
