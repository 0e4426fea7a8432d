"""Cost of channel tracking (oracle/SPEC_KT.md: k_chtrack after the channel detector) on the cfg3 geometry of bench.py.

cfg3 geometry: 296 streams, 65536-point PSD and channeliser, 64 inspectors per stream, 8 channeliser hops (4 PSD
frames) per step, device-resident input, with the channel detector on (k_chdet_fused).  Arms, each built, timed and
released in turn:
  - detector on, tracking off (the launches of an engine without tracking);
  - detector on, tracking on (hold 8) over the cfg3 signal;
  - detector on, tracking on (hold 8) over the cfg3 signal plus a comb of 200 tones, so that at least 200 tracks are
    live whatever the noise does: the most matching work per update (each detection against up to 256 tracks,
    warp-sequential over detections).  The live and dropped counts of stream 0 are reported.
Each step is timed with CUDA events on the engine stream (after the inspector stream has been joined).  A separate
pass in the engine's timing mode gives the device time of the "chan_track" family (one k_chtrack launch per step).
Card name and power limit first.

    python tools/chtrack_rate.py [--streams 296] [--steps 100]
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
    ap.add_argument("--steps", type=int, default=100)
    args = ap.parse_args()
    import numpy as np
    import torch
    import sigdigger_b200 as sdb
    import bench
    if sdb.device_count() < 1:
        raise SystemExit("chtrack_rate.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip())
    bench.FS, bench.N_FFT = 200e6, 65536
    S, N = args.streams, 65536
    n = 8 * N // 2
    base = bench.make_base_signal("cfg3", n, seed=1)
    # 200 tones on exact bins: one detection each
    k = np.arange(n)
    comb = np.zeros(n, np.complex128)
    for i in range(200):
        comb += 0.02 * np.exp(2j * np.pi * ((-32000 + 320 * i + 17) / N * k + i * 0.37))
    dense = (base + comb).astype(np.complex64)

    def signal(b):
        x = torch.from_numpy(b).cuda().unsqueeze(0).repeat(S, 1).contiguous()
        g = torch.Generator(device="cuda").manual_seed(1234)
        x += torch.view_as_complex(1e-3 * torch.randn((S, n, 2), generator=g, device="cuda"))
        return x

    def build(track):
        e = sdb.Engine(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=n, samp_rate=bench.FS)
        for kind, f, baud, bw in bench.workload_channels("cfg3"):
            f0, bwa = bench.chan_angular(f, bw)
            h = e.open_channel(f0, bwa, 1.0)
            cls, kw = bench.insp_kwargs(kind, baud, e.channel_rate(h))
            e.set_inspector(h, cls, **kw)
        e.set_channel_detector(alpha=0.25, beta=0.1, gamma=0.5, snr=4.0, min_bins=2)
        if track:
            e.set_channel_tracking(8)
        e.commit()
        return e

    for name, track, sig in (("detector_only", False, base), ("tracking", True, base), ("tracking_200", True, dense)):
        x = signal(sig)
        e = build(track)
        es = torch.cuda.ExternalStream(e.stream_ptr)

        def step():
            e.feed_device_ptr(x.data_ptr(), x.stride(0), n)

        for _ in range(8):
            step()
        e.sync()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        ev[0].record(es)
        for i in range(args.steps):
            step()
            e.join()
            ev[i + 1].record(es)
        e.sync()
        ms = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(args.steps))
        live = e.read_tracked_channels(0) if track else None
        dets = e.read_channels(0)[1]
        l0 = e.launches
        step()
        e.sync()
        per_step = e.launches - l0
        e.timing(True)
        for _ in range(args.steps):
            step()
        e.sync()
        fam_ms, fam_n = e.kernel_time("chan_track")
        e.timing(False)
        row = dict(arm=name, streams=S, steps=args.steps, launches_per_step=per_step,
                   mean_step_ms=round(sum(ms) / len(ms), 4), median_step_ms=round(ms[len(ms) // 2], 4),
                   gsps=round(S * n / (sum(ms) / len(ms) * 1e-3) / 1e9, 2),
                   detections_stream0=dets, live_tracks_stream0=live[1] if live else None,
                   dropped_stream0=live[2] if live else None,
                   chan_track_ms_per_launch=round(fam_ms, 4), chan_track_launches=fam_n)
        print(json.dumps(row), flush=True)
        e.close()
        del x
        torch.cuda.synchronize()


if __name__ == "__main__":
    main()
