"""Throughput of the stand-alone source decimator (SPEC L, k_decimate) on one GPU, at a batch that fills the card.

For D in {2, 8, 64, 256} and u8 / s16 / f32 input: S streams x n input samples per feed, timed with CUDA events on the
decimator's stream after warm-up.  Each row reports the input rate, the HBM bytes the feed needs (input, plus 8 B per
output) over the 3.35 TB/s data-sheet bandwidth, and the FMAs it needs (2 (16 D + 1) per output) over the FP32
data-sheet rate (67 TFLOP/s = 33.5 T FMA/s), and names the larger of the two as the bound.  Both peaks are data-sheet
figures for an H100 SXM at 700 W; neither is a measurement.

    python tools/decim_rate.py [--streams 296] [--log2n 22] [--reps 7]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
FMA = 33.5e12
BYTES = {"u8": 2, "s16": 4, "f32": 8}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=296)
    ap.add_argument("--log2n", type=int, default=22)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import numpy as np
    import torch
    import sigdigger_b200 as sdb
    if sdb.device_count() < 1:
        raise SystemExit("decim_rate.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip())
    S, n = args.streams, 1 << args.log2n
    g = torch.Generator(device="cuda").manual_seed(1)
    rows = []
    for fmt in ("u8", "s16", "f32"):
        if fmt == "u8":
            x = torch.randint(0, 256, (S, 2 * n), dtype=torch.uint8, device="cuda", generator=g)
        elif fmt == "s16":
            x = torch.randint(-32768, 32768, (S, 2 * n), dtype=torch.int16, device="cuda", generator=g)
        else:
            x = torch.randn(S, n, dtype=torch.complex64, device="cuda", generator=g)
        torch.cuda.synchronize()
        for D in (2, 8, 64, 256):
            dec = sdb.Decimator(D, n_streams=S, input_format=fmt, max_feed=n)
            st = torch.cuda.ExternalStream(dec.stream_ptr)
            times = []
            for r in range(args.warmup + args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                k = dec.feed_ptr(x.data_ptr(), n)
                e1.record(st)
                dec.sync()
                if r >= args.warmup:
                    times.append(e0.elapsed_time(e1) * 1e-3)
            dec.close()
            t_min, t_med = min(times), float(np.median(times))
            byt = S * (n * BYTES[fmt] + k * 8)
            fma = S * k * 2 * (16 * D + 1)
            hbm_share, fma_share = byt / t_min / HBM, fma / t_min / FMA
            row = dict(D=D, fmt=fmt, streams=S, n=n, min_ms=round(t_min * 1e3, 3), median_ms=round(t_med * 1e3, 3),
                       input_gsps=round(S * n / t_min / 1e9, 1), hbm_share=round(hbm_share, 3),
                       fma_share=round(fma_share, 3),
                       bound="HBM" if byt / HBM >= fma / FMA else "FP32")
            rows.append(row)
            print(json.dumps(row), flush=True)
        del x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
