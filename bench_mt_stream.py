"""Streaming multitaper spectrogram through a device MTSpectrogramStream against one call over the whole matrix, on one GPU.

Workloads (each channel a column of a device-resident column-major matrix; dpss tapers, nw = 4, 7 tapers):
  * C4:  64 ch x 2^22 Float32, n = nfft = 1024, 75 % overlap (the bench_mt_channels.py workload; the warp-per-unit
         1024-point plan);
  * cx:  8 ch x 2^22 ComplexF32, n = nfft = 4096, 50 % overlap;
  * fft: 64 ch x 2^22 Float32, n = nfft = 1000 (a cuFFT size: every taper through cuFFT, then added), 75 % overlap.
For each workload and block length C (4096 and 65536 samples per channel) three forms are timed:
  * one_shot: dspb200_mt_spectrogram_batch_exec_dev over the whole matrix (dsp.mt_spectrogram's plan call, into a
    preallocated output);
  * streamed: a device MTSpectrogramStream fed consecutive C x nchan blocks through mt_spectrogram_ into preallocated
    buffers, front end included;
  * launches: the same block sequence through dspb200_stft_stream_exec_dev with every argument precomputed (the device work
    alone).
Times are CUDA events around each form after warm-up, the median of alternating rounds.  In the same run the streamed
columns are checked bit for bit against the one-shot columns.  Prints one JSON line per (workload, block length) with the
card name and power limit.  Writes nothing unless --out is given.
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

WORKLOADS = {"C4": (64, np.float32, 1024, 768), "cx": (8, np.complex64, 4096, 2048), "fft": (64, np.float32, 1000, 750)}
NW = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=22)
    ap.add_argument("--chunks", default="4096,65536")
    ap.add_argument("--workloads", default="C4,cx,fft")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    from dspb200.periodograms import stft_stream_step
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_mt_stream.py needs a CUDA device")
    gpu = card()
    n = 1 << args.log2n

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
        nch, dt, seg, nov = WORKLOADS[name]
        dt = np.dtype(dt)
        rng = np.random.default_rng(2024)
        x = rng.standard_normal((n, nch)).astype(np.float32)
        if dt.kind == "c":
            x = (x + 1j * rng.standard_normal((n, nch)).astype(np.float32)).astype(dt)
        x = np.asfortranarray(x)
        X = dsp.to_device(x)
        cfg = dsp.MTConfig(dt, seg, nfft=seg, nw=NW, noverlap=nov)
        plan1 = cfg.plan
        k = dsp.arraysplit_count(n, seg, nov)
        Y1 = dsp.DeviceArray((plan1.nout, k, nch), np.float32)

        def one_shot():
            plan1.mt_spectrogram_batch_dev(X.ptr, n, nch, Y1.ptr, 0)

        for c in (int(v) for v in args.chunks.split(",")):
            nblk = n // c
            xb = np.concatenate([np.asfortranarray(x[b * c:(b + 1) * c]).ravel(order="F") for b in range(nblk)])
            XB = dsp.to_device(xb)
            isz = dt.itemsize
            xin = [dsp.DeviceArray((c, nch), dt, _base=XB, _ptr=XB.ptr + b * c * nch * isz) for b in range(nblk)]
            s = dsp.MTSpectrogramStream(cfg, nov, device=True)
            h, kcs = 0, []
            for _ in range(nblk):
                kc, h = stft_stream_step(h, c, seg, nov, dt.kind != "c")
                kcs.append(kc)
            kcs.append(stft_stream_step(h, 0, seg, nov, dt.kind != "c", final=True)[0])      # finish()
            offs = np.concatenate([[0], np.cumsum(kcs)])
            YB = dsp.DeviceArray((plan1.nout * int(offs[-1]) * nch,), np.float32)   # block b: its own nout x kc x nch matrix
            outs = [dsp.DeviceArray((plan1.nout, kc, nch), np.float32, _base=YB, _ptr=YB.ptr + int(o) * plan1.nout * nch * 4)
                    for kc, o in zip(kcs, offs)]

            fin = [None]

            def streamed():
                s.reset()
                for b in range(nblk):
                    s.mt_spectrogram_(outs[b], xin[b])
                fin[0] = s.finish().power

            ldh = seg - 1 + (0 if dt.kind == "c" else seg - nov)
            hist = [dsp.DeviceArray((ldh, nch), dt), dsp.DeviceArray((ldh, nch), dt)]
            calls, h = [], 0
            for b in range(nblk + 1):
                nx = c if b < nblk else 0
                hin = None if b == 0 else hist[(b - 1) % 2].ptr
                calls.append((hin, h, hist[b % 2].ptr, ldh, xin[b].ptr if b < nblk else None, nx, nch, kcs[b], 1.0, True,
                              outs[b].ptr, kcs[b], 0))
                h = h + nx - kcs[b] * (seg - nov)

            def launches():
                for a in calls:
                    if a[5] or a[7]:
                        plan1.stft_stream_dev(*a)

            for _ in range(args.warmup):
                one_shot(); streamed(); launches()
            t = {"one_shot": [], "streamed": [], "launches": []}
            for _ in range(args.reps):
                t["one_shot"].append(timed(one_shot))
                t["streamed"].append(timed(streamed))
                t["launches"].append(timed(launches))
            # this run's columns: the stream's concatenation against the one-shot matrix, bit for bit
            l0 = dsp.launch_count()
            streamed()
            torch.cuda.synchronize()
            nlaunch = dsp.launch_count() - l0
            one_shot()
            y1 = Y1.to_host()
            yb = YB.to_host().ravel(order="F")
            ys = np.concatenate([yb[int(o) * plan1.nout * nch:int(o + kc) * plan1.nout * nch].reshape((plan1.nout, kc, nch), order="F")
                                 for kc, o in zip(kcs[:-1], offs)] + [fin[0].to_host()], axis=1)
            launches()
            res = {"workload": f"{name}: {nch} ch x 2^{args.log2n} {dt.name}, n = nfft = {seg}, noverlap {nov}, dpss nw = {NW}, "
                               f"{cfg.ntapers} tapers, MTSpectrogramStream in blocks of {c}",
                   "blocks": nblk, "columns_per_channel": k, "launches_per_stream": nlaunch,
                   "bit_equal_streamed_vs_one_shot": bool(ys.shape == y1.shape and np.array_equal(ys, y1)),
                   "bit_equal_launches_vs_streamed": bool(np.array_equal(YB.to_host().ravel(order="F"), yb))}
            for key, v in t.items():
                ms = float(np.median(v))
                res[key] = {"ms": round(ms, 4), "ms_min": round(float(np.min(v)), 4), "gsamples_per_s": round(n * nch / ms / 1e6, 2)}
            res["streamed_over_one_shot"] = round(res["streamed"]["ms"] / res["one_shot"]["ms"], 3)
            res["launches_over_one_shot"] = round(res["launches"]["ms"] / res["one_shot"]["ms"], 3)
            res["extra_us_per_block_launches"] = round((res["launches"]["ms"] - res["one_shot"]["ms"]) * 1e3 / nblk, 2)
            res["gpu"] = gpu
            lines.append(json.dumps(res))
            print(lines[-1], flush=True)
            del XB, YB, xin, outs, hist
        del X, Y1
        del cfg, plan1
    if args.out:
        with open(args.out, "w") as fo:
            fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
