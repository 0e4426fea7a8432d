"""Cost of the frame-averaged main PSD (SPEC A, k_psd_group_mean) on the cfg3 engine of bench.py.

cfg3 geometry: 296 streams, 65536-point PSD and channeliser, 64 inspectors per stream, 4 PSD frames per stream per step,
device-resident input.  Engines with psd_average = off, 4 and 64 are built side by side and timed in alternating runs
(CUDA events on the engine stream around `--steps` steps, as bench.py times them).  A separate pass in the engine's
timing mode gives the device time of the `psd_average` kernel family per step.  Each row also gives the bytes a caller
reads back per step: the per-frame PSD without averaging, the means with it.  Card name and power limit first.

    python tools/psd_average_rate.py [--streams 296] [--steps 20] [--runs 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=296)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    import sigdigger_b200 as sdb
    import bench
    if sdb.device_count() < 1:
        raise SystemExit("psd_average_rate.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip())
    bench.FS, bench.N_FFT = 200e6, 65536
    S, N = args.streams, 65536
    n = 8 * N // 2                                             # bench.py's 8 hops per step: 4 frames per stream
    base = torch.from_numpy(bench.make_base_signal("cfg3", n, seed=1)).cuda()
    x = base.unsqueeze(0).repeat(S, 1).contiguous()
    g = torch.Generator(device="cuda").manual_seed(1234)
    x += torch.view_as_complex(1e-3 * torch.randn((S, n, 2), generator=g, device="cuda"))
    torch.cuda.synchronize()

    def build(A):
        e = sdb.Engine(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=n, samp_rate=bench.FS,
                       psd_average=A)
        for kind, f, baud, bw in bench.workload_channels("cfg3"):
            f0, bwa = bench.chan_angular(f, bw)
            h = e.open_channel(f0, bwa, 1.0)
            cls, kw = bench.insp_kwargs(kind, baud, e.channel_rate(h))
            e.set_inspector(h, cls, **kw)
        e.commit()
        return e

    arms = {A: build(A) for A in (0, 4, 64)}

    def step(e):
        e.feed_device_ptr(x.data_ptr(), x.stride(0), n)

    def timed(e):
        es = torch.cuda.ExternalStream(e.stream_ptr)
        for _ in range(3):
            step(e)
        e.sync()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(es)
        for _ in range(args.steps):
            step(e)
        e.join()
        b.record(es)
        e.sync()
        return a.elapsed_time(b) / args.steps

    ms = {A: [] for A in arms}
    for _ in range(args.runs):
        for A, e in arms.items():
            ms[A].append(timed(e))
    for A, e in arms.items():
        e.timing(True)
        for _ in range(args.steps):
            step(e)
        e.sync()
        fam_ms, fam_n = e.kernel_time("psd_average")
        e.timing(False)
        # means per step: 4 frames per stream, so a group of A frames completes every A / 4 steps
        read_floats = S * (4 if A < 2 else 4 / A) * N
        row = dict(psd_average=A or "off", streams=S, samples_per_step=S * n,
                   ms_per_step=[round(v, 3) for v in ms[A]],
                   gsps=[round(S * n / (v * 1e-3) / 1e9, 2) for v in ms[A]],
                   psd_average_ms_per_step=round(fam_ms * fam_n / args.steps, 4), psd_average_launches=fam_n,
                   psd_average_read_bytes=S * 4 * N * 4 if A >= 2 else 0,
                   readback_bytes_per_step=int(read_floats * 4))
        print(json.dumps(row), flush=True)
        e.close()


if __name__ == "__main__":
    main()
