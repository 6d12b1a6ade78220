"""Streaming resampling through a device-resident FIRFilter against one call over the whole signal, on one GPU.

Workload: a 64-channel Float32 signal of 2^20 samples per channel in device memory, resampled by 3//2 and by 0.98 with the
default taps (resample_filter: Float64 taps, so the outputs are Float64).  For each rate and block length C (4096 and
65536 samples per channel) three forms are timed:
  * one_shot:     a fresh device FIRFilter (reset()) given the whole 2^20 x 64 matrix as one chunk;
  * streamed:     the same filter fed consecutive C x 64 column-major blocks through filt_ into preallocated buffers, as an
                  acquisition would deliver them; this includes the Python front end's work for every block;
  * launches:     the same blocks through the C ABI (ResamplePlan.stream_exec_dev) with every argument precomputed, so
                  the difference to `streamed` is the front end's host cost and this one is the device work.
A block costs two launches: the outputs whose window reaches into the previous block (about H*I/D per channel, H = taps per
phase - 1) with the new history, then the rest.  Times are CUDA events around each form (device-resident inputs, no copies),
after warm-up, the forms alternating.  In the same run the outputs are checked: at 3//2 the streamed outputs must equal the
one-shot output bit for bit; at 0.98 every call restarts from a rounded phase accumulator, so there the streamed output must
equal a host FIRFilter streamed in the same blocks on two channels bit for bit, and the one-shot output within 2e-6.

Prints one JSON line per (rate, block length) with the card name and power limit.  Writes nothing unless --out is given.
"""
import argparse
import json
import os
import sys
from fractions import Fraction

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_fir_stream import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=64)
    ap.add_argument("--log2n", type=int, default=20)
    ap.add_argument("--chunks", default="4096,65536")
    ap.add_argument("--rates", default="3//2,0.98")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch
    import dspb200 as dsp
    if not torch.cuda.is_available() or dsp.device_count() < 1:
        raise SystemExit("bench_resample_stream.py needs a CUDA device")
    gpu = card()
    nch, n = args.channels, 1 << args.log2n
    x = np.random.default_rng(2024).standard_normal((n, nch)).astype(np.float32)
    X = dsp.to_device(x)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    lines = []
    for rtxt in args.rates.split(","):
        arb = "//" not in rtxt
        rate = float(rtxt) if arb else Fraction(rtxt.replace("//", "/"))
        h = dsp.resample_filter(rate)
        f1 = dsp.FIRFilter(h, rate, device=True)
        nout1 = f1._step(1, 1, 0.0, n).nout
        Y1 = dsp.DeviceArray((nout1, nch), np.float64)

        def one_shot():
            f1.reset()
            dsp.filt_(Y1, f1, X)

        for c in (int(v) for v in args.chunks.split(",")):
            if n % c:
                raise SystemExit(f"block length {c} must divide {n}")
            nblk = n // c
            xb = np.concatenate([np.asfortranarray(x[k * c:(k + 1) * c]).ravel(order="F") for k in range(nblk)])
            XB = dsp.to_device(xb)
            xin = [dsp.DeviceArray((c, nch), np.float32, _base=XB, _ptr=XB.ptr + k * c * nch * 4) for k in range(nblk)]
            # per-block bookkeeping of a fresh filter: output counts and the arguments of every C ABI call
            f = dsp.FIRFilter(h, rate, device=True)
            steps, s = [], (f.phi_idx, f.input_deficit, f.phi_accumulator)
            for _ in range(nblk):
                st = f._step(*s, c)
                steps.append((s[1], st))
                s = (st.phi_idx, st.input_deficit, st.phi_accumulator)
            rows = [st.nout for _, st in steps]
            offs = np.concatenate([[0], np.cumsum(rows)]) * nch * 8
            YB = dsp.DeviceArray((int(offs[-1]) // 8,), np.float64)
            yout = [dsp.DeviceArray((r, nch), np.float64, _base=YB, _ptr=YB.ptr + int(o)) for r, o in zip(rows, offs)]

            def streamed():
                f.reset()
                for k in range(nblk):
                    dsp.filt_(yout[k], f, xin[k])

            plan = f._plan(np.dtype(np.float32))
            H = f.history_len
            hist = [dsp.DeviceArray((H, nch), np.float32), dsp.DeviceArray((H, nch), np.float32)]
            calls = []
            for k, (deficit, st) in enumerate(steps):
                hin = None if k == 0 else hist[(k - 1) % 2].ptr
                a = (hin, hist[k % 2].ptr, xin[k].ptr, c, nch, deficit, st.phase0)
                calls.append(a + ((f.delta,) if arb else ()) + (yout[k].ptr, st.nout, st.nout, 0))

            def launches():
                for a in calls:
                    plan.stream_exec_dev(*a)

            for _ in range(args.warmup):
                one_shot(); streamed(); launches()
            t = {"one_shot": [], "streamed": [], "launches": []}
            for _ in range(args.reps):
                t["one_shot"].append(timed(one_shot))
                t["streamed"].append(timed(streamed))
                t["launches"].append(timed(launches))
            # outputs of this run: streamed (through filt_) against one-shot, and at 0.98 against the host form
            l0 = dsp.launch_count()
            streamed()
            nlaunch = dsp.launch_count() - l0
            one_shot()
            yb = YB.to_host()
            ys = np.concatenate([yb[int(o) // 8:int(o) // 8 + r * nch].reshape(nch, r).T for r, o in zip(rows, offs)])
            y1 = Y1.to_host()
            res = {"workload": f"{nch} ch x 2^{args.log2n} Float32, rate {rtxt}, {h.size} Float64 taps, device FIRFilter "
                               f"in blocks of {c}",
                   "blocks": nblk, "launches_per_stream": nlaunch, "seam_outputs_per_block": steps[1][1].j_seam if nblk > 1 else 0}
            launches()
            launched_equal = bool(np.array_equal(YB.to_host(), yb))
            if arb:
                hosts = {cc: dsp.FIRFilter(h, rate) for cc in (0, nch - 1)}
                hs = {cc: np.concatenate([g.filt(x[k * c:(k + 1) * c, cc]) for k in range(nblk)]) for cc, g in hosts.items()}
                res["bit_equal_streamed_vs_host_streamed"] = bool(all(np.array_equal(ys[:, cc], v) for cc, v in hs.items()))
                m = min(ys.shape[0], y1.shape[0])
                res["max_rel_diff_streamed_vs_one_shot"] = float(np.max(np.abs(ys[:m] - y1[:m])) / np.max(np.abs(y1[:m])))
                res["within_2e-6_of_one_shot"] = res["max_rel_diff_streamed_vs_one_shot"] <= 2e-6
            else:
                res["bit_equal_streamed_vs_one_shot"] = bool(ys.shape == y1.shape and np.array_equal(ys, y1))
            res["bit_equal_launches_vs_streamed"] = launched_equal
            for key, v in t.items():
                ms = float(np.median(v))
                res[key] = {"ms": round(ms, 4), "ms_min": round(float(np.min(v)), 4), "gsamples_per_s": round(n * nch / ms / 1e6, 2)}
            res["streamed_over_one_shot"] = round(res["streamed"]["ms"] / res["one_shot"]["ms"], 3)
            res["launches_over_one_shot"] = round(res["launches"]["ms"] / res["one_shot"]["ms"], 3)
            res["gpu"] = gpu
            lines.append(json.dumps(res))
            print(lines[-1], flush=True)
            del XB, YB, xin, yout, hist
    if args.out:
        with open(args.out, "w") as fo:
            fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
