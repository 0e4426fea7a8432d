"""Cost of the inspector's Analog TV tab (oracle/SPEC_TI.md, k_tv_insp in tv_kernels.cu) on the cfg3 engine of
bench.py.

cfg3 geometry: 296 streams, 65536-point PSD and channeliser, 64 inspectors per stream, 8 hops per step, device-resident
input.  The TV runs on a subset of the psk / fsk / ask inspectors with the PAL picture of an 8 MS/s signal (W 512,
H 625: 6.4 MB per stream, about 1.9 GB per inspector over 296 streams), fed at each inspector's own symbol rate.  Three
plans are built side by side in the same call: the stock plan (TV off), the TV on 1 inspector and on --many
inspectors.  Step times come from CUDA events on the engine stream around `--steps` steps (as bench.py times them), in
alternating runs; a separate pass in the engine's timing mode gives the device time of the "tv" kernel family per
step, and the symbols the TV processors took in that step give the serial step's cost per symbol.  Card name, power
limit and clock first.

    python tools/tv_rate.py [--streams 296] [--steps 20] [--runs 3] [--many 8]
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
    ap.add_argument("--many", type=int, default=8)
    args = ap.parse_args()
    import torch
    import sigdigger_b200 as sdb
    import bench
    if sdb.device_count() < 1:
        raise SystemExit("tv_rate.py needs a CUDA device")
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
    pal = sdb.tv_params("pal", 8e6)

    def build(k_tv):
        e = sdb.Engine(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=n, samp_rate=bench.FS)
        tv = []
        for kind, f, baud, bw in chans:
            f0, bwa = bench.chan_angular(f, bw)
            h = e.open_channel(f0, bwa, 1.0)
            cls, kw = bench.insp_kwargs(kind, baud, e.channel_rate(h))
            e.set_inspector(h, cls, **kw)
            if len(tv) < k_tv and cls in ("psk", "fsk", "ask"):
                e.set_tv(h, params=pal)
                tv.append(h)
        e.commit()
        return e, tv

    arms = {}
    for k in (0, 1, args.many):
        arms[k] = build(k)

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

    ms = {k: [] for k in arms}
    for _ in range(args.runs):
        for k, (e, _) in arms.items():
            ms[k].append(timed(e))
    for k, (e, tv) in arms.items():
        e.timing(True)
        for _ in range(args.steps):
            step(e)
        e.sync()
        tv_ms, tv_n = e.kernel_time("tv")
        in_ms, in_n = e.kernel_time("inspector")
        e.timing(False)
        # symbols one step hands to the TV processors: every stream of a channel carries the same signal, so stream 0
        # stands for all; the longest processor bounds the launch (one warp each, serial in its symbols)
        per_proc = [len(e.read_symbols(0, h)[0]) for h in tv]
        row = dict(tv_channels=len(tv), streams=S, tv_processors=len(tv) * S, samples_per_step=S * n,
                   ms_per_step=[round(v, 3) for v in ms[k]], gsps=[round(S * n / (v * 1e-3) / 1e9, 2) for v in ms[k]],
                   tv_ms_per_step=round(tv_ms * tv_n / args.steps, 4), tv_launches=tv_n,
                   inspector_ms_per_step=round(in_ms * in_n / args.steps, 4),
                   symbols_per_processor_step=per_proc, launches=e.launches)
        if tv and tv_n and max(per_proc):
            row["ns_per_symbol_longest_processor"] = round(tv_ms * 1e6 / max(per_proc), 2)
        print(json.dumps(row), flush=True)
        e.close()


if __name__ == "__main__":
    main()
