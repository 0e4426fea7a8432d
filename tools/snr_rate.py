"""Cost of the inspector's SNR meter (oracle/SPEC_SN.md, snr_kernels.cu) on the cfg3 engine of bench.py.

cfg3 geometry: 296 streams, 65536-point PSD and channeliser, 64 inspectors per stream, 8 hops per step,
device-resident input.  Three plans are built side by side in the same call: the stock plan (meter off), and the meter
on every psk / fsk / ask inspector at L = 256 (the GUI's histogram) and at L = 1024, with the GUI's toggle values
(sigma 1, alpha 1 / 2^bps).  Step times come from CUDA events on the engine stream around `--steps` steps (as bench.py
times them), in alternating runs; a separate pass in the engine's timing mode gives the device time of the "snr"
kernel family per step.  Card name and power limit first.

    python tools/snr_rate.py [--streams 296] [--steps 20] [--runs 3]
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
    import torch
    import sigdigger_b200 as sdb
    import bench
    if sdb.device_count() < 1:
        raise SystemExit("snr_rate.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip())
    bench.FS, bench.N_FFT = 200e6, 65536
    S, N = args.streams, 65536
    n = 8 * N // 2                                             # bench.py's 8 hops per step
    base = torch.from_numpy(bench.make_base_signal("cfg3", n, seed=1)).cuda()
    x = base.unsqueeze(0).repeat(S, 1).contiguous()
    g = torch.Generator(device="cuda").manual_seed(1234)
    x += torch.view_as_complex(1e-3 * torch.randn((S, n, 2), generator=g, device="cuda"))
    torch.cuda.synchronize()
    chans = bench.workload_channels("cfg3")

    def build(L):
        e = sdb.Engine(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=n, samp_rate=bench.FS)
        n_snr = 0
        for kind, f, baud, bw in chans:
            f0, bwa = bench.chan_angular(f, bw)
            h = e.open_channel(f0, bwa, 1.0)
            cls, kw = bench.insp_kwargs(kind, baud, e.channel_rate(h))
            e.set_inspector(h, cls, **kw)
            if L and cls in ("psk", "fsk", "ask"):
                e.set_snr(h, bins=L)
                n_snr += 1
        e.commit()
        return e, n_snr

    arms = {}
    for L in (0, 256, 1024):
        arms[L] = build(L)

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

    ms = {L: [] for L in arms}
    for _ in range(args.runs):
        for L, (e, _) in arms.items():
            ms[L].append(timed(e))
    for L, (e, n_snr) in arms.items():
        e.timing(True)
        for _ in range(args.steps):
            step(e)
        e.sync()
        snr_ms, snr_n = e.kernel_time("snr")
        in_ms, in_n = e.kernel_time("inspector")
        e.timing(False)
        row = dict(snr_bins=L or None, streams=S, snr_channels=n_snr, snr_chains=n_snr * S,
                   samples_per_step=S * n, ms_per_step=[round(v, 3) for v in ms[L]],
                   gsps=[round(S * n / (v * 1e-3) / 1e9, 2) for v in ms[L]],
                   snr_ms_per_step=round(snr_ms * snr_n / args.steps, 4), snr_launches=snr_n,
                   inspector_ms_per_step=round(in_ms * in_n / args.steps, 4), launches=e.launches)
        print(json.dumps(row), flush=True)
        e.close()


if __name__ == "__main__":
    main()
