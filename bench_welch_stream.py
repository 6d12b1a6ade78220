"""Streaming Welch through a device WelchStream against one batched welch_pgram over the whole matrix, on one GPU.

Workloads (each channel a column of a device-resident column-major matrix, seeded):
  * real: 64 ch x 2^22 Float32, n = nfft = 4096, 50 % overlap, hanning (the fused two-for-one real kernel);
  * cx:   8 ch x 2^24 ComplexF32, n = nfft = 4096, 50 % overlap, hanning (the fused complex kernel);
  * fft:  64 ch x 2^20 Float32, n = nfft = 1000 (a cuFFT size), 50 % overlap, hanning.
For each workload and block length C (4096 and 65536 samples per channel) three forms are timed:
  * one_shot: dspb200_welch_batch_exec_dev over the whole matrix (welch_pgram's batched plan call, into a preallocated output);
  * streamed: a device WelchStream fed consecutive C x nchan blocks through update(), then welch_pgram_ into a preallocated
    output, front end included;
  * launches: the same block sequence and power read through the C ABI with every argument precomputed (the device work alone).
Times are CUDA events around each form after warm-up, the median of alternating rounds.  In the same run: the power of a
stream given the whole matrix as one chunk against the one-shot power, bit for bit (promised for fused sizes), and the
largest per-bin relative difference of the block-streamed power from the one-shot power.  Prints one JSON line per
(workload, block length) with the card name and power limit.  Writes nothing unless --out is given.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_fir_stream import card  # noqa: E402

WORKLOADS = {"real": (64, 22, np.float32, 4096, 2048), "cx": (8, 24, np.complex64, 4096, 2048),
             "fft": (64, 20, np.float32, 1000, 500)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", default="4096,65536")
    ap.add_argument("--workloads", default="real,cx,fft")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    from dspb200 import _lib
    from dspb200.periodograms import stft_stream_step
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_welch_stream.py needs a CUDA device")
    gpu = card()

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    lines = []
    for name in args.workloads.split(","):
        nch, log2n, dt, seg, nov = WORKLOADS[name]
        n = 1 << log2n
        dt = np.dtype(dt)
        rng = np.random.default_rng(2024)
        x = rng.standard_normal((n, nch)).astype(np.float32)
        if dt.kind == "c":
            x = (x + 1j * rng.standard_normal((n, nch)).astype(np.float32)).astype(dt)
        x = np.asfortranarray(x)
        X = dsp.to_device(x)
        win, norm2 = dsp.compute_window(dsp.hanning, seg)
        plan1 = _lib.SpecPlan(dt, seg, nov, seg, dt.kind != "c", win)
        k = dsp.arraysplit_count(n, seg, nov)
        P1 = dsp.DeviceArray((plan1.nout, nch), np.float32)

        def one_shot():
            plan1.welch_batch_dev(X.ptr, n, nch, k * norm2, P1.ptr, 0)

        # one chunk from an empty history: the one-shot power, bit for bit (fused sizes)
        s1 = dsp.WelchStream(seg, nov, nfft=seg, window=dsp.hanning, device=True)
        s1.update(X)
        one_chunk = s1.welch_pgram().power.to_host()
        one_shot()
        p1 = P1.to_host()
        del s1

        for c in (int(v) for v in args.chunks.split(",")):
            nblk = n // c
            xb = np.concatenate([np.asfortranarray(x[b * c:(b + 1) * c]).ravel(order="F") for b in range(nblk)])
            XB = dsp.to_device(xb)
            del xb
            isz = dt.itemsize
            xin = [dsp.DeviceArray((c, nch), dt, _base=XB, _ptr=XB.ptr + b * c * nch * isz) for b in range(nblk)]
            s = dsp.WelchStream(seg, nov, nfft=seg, window=dsp.hanning, device=True)
            PS = dsp.DeviceArray((plan1.nout, nch), np.float32)

            def streamed():
                s.reset()
                for b in range(nblk):
                    s.update(xin[b])
                s.welch_pgram_(PS)

            plan2 = _lib.SpecPlan(dt, seg, nov, seg, dt.kind != "c", win)
            ldh = seg - 1
            hist = [dsp.DeviceArray((ldh, nch), dt), dsp.DeviceArray((ldh, nch), dt)]
            acc = dsp.DeviceArray((plan2.nout, nch), np.float64)
            PL = dsp.DeviceArray((plan2.nout, nch), np.float32)
            calls, h, tot = [], 0, 0
            for b in range(nblk):
                kc, newh = stft_stream_step(h, c, seg, nov, False)
                calls.append((None if b == 0 else hist[(b - 1) % 2].ptr, h, hist[b % 2].ptr, ldh, xin[b].ptr, c, nch, kc,
                              acc.ptr, tot > 0, 0))
                h, tot = newh, tot + kc

            def launches():
                for a in calls:
                    plan2.welch_stream_dev(*a)
                plan2.welch_stream_power_dev(acc.ptr, nch, tot * norm2, PL.ptr, 0)

            for _ in range(args.warmup):
                one_shot(); streamed(); launches()
            t = {"one_shot": [], "streamed": [], "launches": []}
            for _ in range(args.reps):
                t["one_shot"].append(timed(one_shot))
                t["streamed"].append(timed(streamed))
                t["launches"].append(timed(launches))
            l0 = dsp.launch_count()
            streamed()
            torch.cuda.synchronize()
            nlaunch = dsp.launch_count() - l0
            ps = PS.to_host()
            launches()
            pl = PL.to_host()
            rel = np.abs(ps.astype(np.float64) - p1) / np.maximum(np.abs(p1.astype(np.float64)), 1e-300)
            res = {"workload": f"{name}: {nch} ch x 2^{log2n} {dt.name}, n = nfft = {seg}, noverlap {nov}, hanning, "
                               f"WelchStream in blocks of {c}",
                   "blocks": nblk, "segments_per_channel": k, "segments_streamed": s.nsegments,
                   "launches_per_stream": nlaunch,
                   "bit_equal_one_chunk_vs_one_shot": bool(np.array_equal(one_chunk, p1)),
                   "max_rel_diff_streamed_vs_one_shot": float(rel.max()),
                   "bit_equal_launches_vs_streamed": bool(np.array_equal(pl, ps))}
            for key, v in t.items():
                ms = float(np.median(v))
                res[key] = {"ms": round(ms, 4), "ms_min": round(float(np.min(v)), 4), "gsamples_per_s": round(n * nch / ms / 1e6, 2)}
            res["streamed_over_one_shot"] = round(res["streamed"]["ms"] / res["one_shot"]["ms"], 3)
            res["launches_over_one_shot"] = round(res["launches"]["ms"] / res["one_shot"]["ms"], 3)
            res["extra_us_per_block_launches"] = round((res["launches"]["ms"] - res["one_shot"]["ms"]) * 1e3 / nblk, 2)
            res["gpu"] = gpu
            lines.append(json.dumps(res))
            print(lines[-1], flush=True)
            del XB, xin, hist, acc, PS, PL
            plan2.close()
        del X, P1
        plan1.close()
    if args.out:
        with open(args.out, "w") as fo:
            fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
