"""Cost of the power inspector (SPEC PW, k_power_integrate) on the cfg3 engine of bench.py.

cfg3 geometry: 296 streams, 65536-point PSD and channeliser, 64 inspectors per stream, 8 hops per step, device-resident
input.  Three plans are built side by side: the stock cfg3 plan, the same plan with one power channel added, and the
cfg3 channels with every inspector a power inspector.  Step times come from CUDA events on the engine stream around
`--steps` steps (as bench.py times them), in alternating runs; a separate pass in the engine's timing mode gives the
device time of the `power` kernel family per step.  Card name and power limit first.

    python tools/power_rate.py [--streams 296] [--steps 20] [--runs 3] [--M 100000]
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
    ap.add_argument("--M", type=int, default=100000, help="power.integrate-samples of every power inspector")
    args = ap.parse_args()
    import torch
    import sigdigger_b200 as sdb
    import bench
    if sdb.device_count() < 1:
        raise SystemExit("power_rate.py needs a CUDA device")
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

    def build(plan):
        e = sdb.Engine(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=n, samp_rate=bench.FS)
        n_power = 0
        for kind, f, baud, bw in chans:
            f0, bwa = bench.chan_angular(f, bw)
            h = e.open_channel(f0, bwa, 1.0)
            if plan == "all_power":
                e.set_inspector(h, "power", power_integrate_samples=args.M)
                n_power += 1
            else:
                cls, kw = bench.insp_kwargs(kind, baud, e.channel_rate(h))
                e.set_inspector(h, cls, **kw)
        if plan == "stock_plus_one":
            kind, f, baud, bw = chans[0]
            f0, bwa = bench.chan_angular(f, bw)
            h = e.open_channel(f0, bwa, 1.0)
            e.set_inspector(h, "power", power_integrate_samples=args.M)
            n_power += 1
        e.commit()
        return e, n_power

    arms = {p: build(p) for p in ("stock", "stock_plus_one", "all_power")}

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

    ms = {p: [] for p in arms}
    for _ in range(args.runs):
        for p, (e, _) in arms.items():
            ms[p].append(timed(e))
    for p, (e, n_power) in arms.items():
        e.timing(True)
        for _ in range(args.steps):
            step(e)
        e.sync()
        pw_ms, pw_n = e.kernel_time("power")
        in_ms, in_n = e.kernel_time("inspector")
        e.timing(False)
        row = dict(plan=p, streams=S, power_channels=n_power, power_chains=n_power * S, M=args.M,
                   samples_per_step=S * n, ms_per_step=[round(v, 3) for v in ms[p]],
                   gsps=[round(S * n / (v * 1e-3) / 1e9, 2) for v in ms[p]],
                   power_ms_per_step=round(pw_ms * pw_n / args.steps, 4), power_launches=pw_n,
                   inspector_ms_per_step=round(in_ms * in_n / args.steps, 4))
        print(json.dumps(row), flush=True)
        e.close()


if __name__ == "__main__":
    main()
