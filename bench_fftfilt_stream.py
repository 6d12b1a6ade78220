"""Streaming a DF2TFilter by overlap-save (fftfilt(f, x)) against the time-domain stream (filt(f, x)) and one stateless
overlap-save call over the whole signal, on one GPU.

Workloads (device-resident seeded inputs, preallocated outputs, no copies):
  * 64 channels x 2^20 Float32 samples, 257 and 4097 taps, in blocks of C = 4096 and 65536 samples x 64 channels (each
    block a column-major C x 64 array); four forms:
      direct    -- a device DF2TFilter fed the blocks through filt_ (time-domain tile kernel, one launch per block);
      fftfilt   -- the same filter through fftfilt_ (stateful overlap-save, one launch per block);
      launches  -- the stateful overlap-save launches alone through the C ABI (dspb200_os_exec_state_dev);
      one_shot  -- one stateless overlap-save call over the whole 2^20 x 64 matrix (dspb200_os_exec_dev);
  * 2^26 ComplexF32 samples, one channel, 4097 taps, in blocks of 2^20 and 2^22: fftfilt against one stateless
    dspb200_os_exec_dev over the whole signal (the headline kernel).
Times are CUDA events around each form, after warm-up, the forms alternating round by round; the median and minimum over
the rounds are reported.  A stream of C-sample blocks computes C + nb - 1 outputs per channel and block (the last nb - 1
are the carried state), so it is expected near the one-shot time plus (nb - 1) / C extra outputs, rounded up to whole
units, plus one launch per block.  In the same run every stream's output is compared with the one-shot output (the largest
absolute difference is reported; the direct and overlap-save streams differ from it by rounding only).

Prints one JSON line per (workload, block) with the card name and power limit.  Writes nothing unless --out is given.
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


def lowpass(nb):
    n = np.arange(nb) - (nb - 1) / 2
    return (0.5 * np.sinc(0.5 * n) * np.hamming(nb)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=64)
    ap.add_argument("--log2n", type=int, default=20)
    ap.add_argument("--taps", default="257,4097")
    ap.add_argument("--chunks", default="4096,65536")
    ap.add_argument("--log2n-complex", type=int, default=26)
    ap.add_argument("--chunks-complex", default="1048576,4194304")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_fftfilt_stream.py needs a CUDA device")
    gpu = card()
    lines = []

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def run(forms, n_total, res):
        for _ in range(args.warmup):
            for fn in forms.values():
                fn()
        t = {k: [] for k in forms}
        for _ in range(args.reps):
            for k, fn in forms.items():
                t[k].append(timed(fn))
        for k, v in t.items():
            ms = float(np.median(v))
            res[k] = {"ms": round(ms, 4), "ms_min": round(float(np.min(v)), 4), "gsamples_per_s": round(n_total / ms / 1e6, 2)}
        res["gpu"] = gpu
        lines.append(json.dumps(res))
        print(lines[-1], flush=True)

    def launches(fn):
        l0 = dsp.launch_count()
        fn()
        torch.cuda.synchronize()
        return dsp.launch_count() - l0

    def stream_forms(dt, b, X, n, nch, c, Y, Yd):
        """Block views of X / Y / Yd and the three streamed forms (direct, fftfilt, launches through the C ABI)."""
        nblk = n // c
        step = c * nch * np.dtype(dt).itemsize
        xin = [dsp.DeviceArray((c, nch), dt, _base=X, _ptr=X.ptr + k * step) for k in range(nblk)]
        yout = [dsp.DeviceArray((c, nch), dt, _base=Y, _ptr=Y.ptr + k * step) for k in range(nblk)]
        ydir = [dsp.DeviceArray((c, nch), dt, _base=Yd, _ptr=Yd.ptr + k * step) for k in range(nblk)] if Yd is not None else None
        pr = dsp.PolynomialRatio(b, np.ones(1, dt))
        st = {"fd": dsp.DF2TFilter(pr, (nch,), device=True), "ff": dsp.DF2TFilter(pr, (nch,), device=True)}
        plan = dsp._lib.OsPlan(b, 0)
        s = [dsp.DeviceArray((b.size - 1, nch), dt), dsp.DeviceArray((b.size - 1, nch), dt)]

        def direct():
            for k in range(nblk):
                dsp.filt_(ydir[k], st["fd"], xin[k])

        def fft():
            for k in range(nblk):
                dsp.fftfilt_(yout[k], st["ff"], xin[k])

        def abi():
            for k in range(nblk):
                plan.exec_state_dev(xin[k].ptr, c, nch, s[k & 1].ptr if k else None, s[(k + 1) & 1].ptr, yout[k].ptr, 0)

        def fresh():
            st["fd"] = dsp.DF2TFilter(pr, (nch,), device=True)
            st["ff"] = dsp.DF2TFilter(pr, (nch,), device=True)
            st["ff"]._os_plan(np.dtype(dt))          # plan (filter transform) now, so the stream counts only its own launches
        return direct, fft, abi, fresh, plan

    def unblock(Yb, n, nch, c):
        """Block-laid output (block k: a c x nch column-major array) -> n x nch."""
        yb = Yb.to_host().reshape(n // c, nch, c)
        return np.ascontiguousarray(yb.transpose(0, 2, 1)).reshape(n, nch)

    # ------------------------------------------------------------------------------------ 64 x 2^20 Float32
    nch, n = args.channels, 1 << args.log2n
    x = np.random.default_rng(2024).standard_normal((n, nch)).astype(np.float32)
    X1 = dsp.to_device(x)
    Y1 = dsp.DeviceArray((n, nch), np.float32)
    for nb in (int(v) for v in args.taps.split(",")):
        b = lowpass(nb)
        one = dsp._lib.OsPlan(b, 0)

        def one_shot():
            one.exec_dev(X1.ptr, n, nch, Y1.ptr, n, 0)
        for c in (int(v) for v in args.chunks.split(",")):
            if n % c:
                raise SystemExit(f"block length {c} must divide {n}")
            xb = np.concatenate([np.asfortranarray(x[k * c:(k + 1) * c]).ravel(order="F") for k in range(n // c)])
            XB = dsp.to_device(xb)
            YB, YD = dsp.DeviceArray(xb.shape, np.float32), dsp.DeviceArray(xb.shape, np.float32)
            direct, fft, abi, fresh, plan = stream_forms(np.float32, b, XB, n, nch, c, YB, YD)
            res = {"workload": f"{nch} ch x 2^{args.log2n} Float32, {nb} taps (nfft {plan.nfft}), DF2TFilter in blocks of {c}",
                   "blocks": n // c, "extra_outputs_fraction": round((nb - 1) / c, 5)}
            fresh()
            res["launches_per_stream"] = {"direct": launches(direct), "launches": launches(abi), "fftfilt": launches(fft),
                                          "one_shot": launches(one_shot)}
            y1 = Y1.to_host()
            res["max_abs_diff_vs_one_shot"] = {"direct": float(np.max(np.abs(unblock(YD, n, nch, c) - y1))),
                                               "fftfilt": float(np.max(np.abs(unblock(YB, n, nch, c) - y1)))}
            run({"direct": direct, "fftfilt": fft, "launches": abi, "one_shot": one_shot}, n * nch, res)
            plan.close()
            del XB, YB, YD
        one.close()
    del X1, Y1

    # ------------------------------------------------------------------------------------ 2^26 ComplexF32, one channel
    n = 1 << args.log2n_complex
    rng = np.random.default_rng(26)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    b = (lowpass(4097) * np.exp(0.3j * np.arange(4097))).astype(np.complex64)
    X = dsp.to_device(x.reshape(n, 1))
    Y1, Y = dsp.DeviceArray((n, 1), np.complex64), dsp.DeviceArray((n, 1), np.complex64)
    one = dsp._lib.OsPlan(b, 0)

    def one_shot_c():
        one.exec_dev(X.ptr, n, 1, Y1.ptr, n, 0)
    for c in (int(v) for v in args.chunks_complex.split(",")):
        _, fft, _, fresh, plan = stream_forms(np.complex64, b, X, n, 1, c, Y, None)
        res = {"workload": f"2^{args.log2n_complex} ComplexF32, 1 ch, 4097 taps (nfft {plan.nfft}), fftfilt in blocks of {c}",
               "blocks": n // c, "extra_outputs_fraction": round(4096 / c, 5)}
        fresh()
        res["launches_per_stream"] = {"fftfilt": launches(fft), "one_shot": launches(one_shot_c)}
        res["max_abs_diff_vs_one_shot"] = {"fftfilt": float(np.max(np.abs(Y.to_host() - Y1.to_host())))}
        run({"fftfilt": fft, "one_shot": one_shot_c}, n, res)
        plan.close()
    one.close()
    if args.out:
        with open(args.out, "w") as fo:
            fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
