"""Cost of the main PSD's frame-group stages on the cfg3 engine of bench.py: the frame-averaged PSD (SPEC A,
k_psd_group_mean) and the peak detectors (SPEC PK, k_psd_group_peak).

cfg3 geometry: 296 streams, 65536-point PSD and channeliser, 64 inspectors per stream, 4 PSD frames per stream per step,
device-resident input.  Six engines are built side by side: both stages off; A = 4 (one mean a step); A = 64; P = 4 (one
group a step); P = 122 (the frames of one 40 ms psd_update_int at 200 MS/s: a group stays open across steps, so the
carry moves every step); and P = 4 with A = 4.  They are timed in alternating runs (CUDA events on the engine stream
around `--steps` steps, as bench.py times them).  A separate pass in the engine's timing mode gives the device time and
launches per step of the `psd_average` and `psd_peak` kernel families.  Each row also gives the bytes a caller reads
back per step (the per-frame PSD without averaging, the means with it) and the bytes k_psd_group_peak moves per step.
Card name and power limit first.

    python tools/psd_group_rate.py [--streams 296] [--steps 20] [--runs 3]
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
        raise SystemExit("psd_group_rate.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip())
    bench.FS, bench.N_FFT = 200e6, 65536
    S, N, F = args.streams, 65536, 4
    n = 8 * N // 2                                             # bench.py's 8 hops per step: 4 frames per stream
    base = torch.from_numpy(bench.make_base_signal("cfg3", n, seed=1)).cuda()
    x = base.unsqueeze(0).repeat(S, 1).contiguous()
    g = torch.Generator(device="cuda").manual_seed(1234)
    x += torch.view_as_complex(1e-3 * torch.randn((S, n, 2), generator=g, device="cuda"))
    torch.cuda.synchronize()

    def build(A, P):
        e = sdb.Engine(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=n, samp_rate=bench.FS,
                       psd_average=A, psd_peak=P)
        for kind, f, baud, bw in bench.workload_channels("cfg3"):
            f0, bwa = bench.chan_angular(f, bw)
            h = e.open_channel(f0, bwa, 1.0)
            cls, kw = bench.insp_kwargs(kind, baud, e.channel_rate(h))
            e.set_inspector(h, cls, **kw)
        e.commit()
        return e

    arms = {(A, P): build(A, P) for A, P in ((0, 0), (4, 0), (64, 0), (0, 4), (0, 122), (4, 4))}

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
        for k, e in arms.items():
            ms[k].append(timed(e))
    for (A, P), e in arms.items():
        e.timing(True)
        for _ in range(args.steps):
            step(e)
        e.sync()
        avg_ms, avg_n = e.kernel_time("psd_average")
        peak_ms, peak_n = e.kernel_time("psd_peak")
        e.timing(False)
        avg_step_ms, peak_step_ms = avg_ms * avg_n / args.steps, peak_ms * peak_n / args.steps
        # means per step: 4 frames per stream, so a group of A frames completes every A / 4 steps
        read_floats = S * (F if A < 2 else F / A) * N
        # bytes of k_psd_group_peak per step: the frames in; per finished group two outputs; with a group open across
        # the step boundary (P = 122) both carries in and out
        groups_per_step = F / P if P >= 2 else 0
        carry = 4 if P >= 2 and P % F else 0
        peak_bytes = int(S * N * 4 * (F + 2 * groups_per_step + carry)) if P >= 2 else 0
        row = dict(psd_average=A or "off", psd_peak=P or "off", streams=S, samples_per_step=S * n,
                   ms_per_step=[round(v, 3) for v in ms[(A, P)]],
                   gsps=[round(S * n / (v * 1e-3) / 1e9, 2) for v in ms[(A, P)]],
                   psd_average_ms_per_step=round(avg_step_ms, 4), psd_average_launches=avg_n,
                   psd_average_read_bytes=S * F * N * 4 if A >= 2 else 0,
                   readback_bytes_per_step=int(read_floats * 4),
                   psd_peak_ms_per_step=round(peak_step_ms, 4), psd_peak_launches=peak_n,
                   psd_peak_bytes_per_step=peak_bytes,
                   psd_peak_gbps=round(peak_bytes / (peak_step_ms * 1e-3) / 1e9, 1) if peak_n else None)
        print(json.dumps(row), flush=True)
        e.close()


if __name__ == "__main__":
    main()
