"""Cost of scheduled inspector spectra (SPEC US: k_spectsched_gather, k_spectsrc over the emitted frames,
k_spectsched_ring) on the cfg3 engine of bench.py.

cfg3 geometry: 296 streams, 65536-point PSD and channeliser, 64 inspectors per stream (1024-bin channels at
3.125 MS/s), 8 channeliser hops per step, so 4096 channel samples per channel per step, device-resident input.  Arms,
each built, timed and released in turn:
  - no spectrum source (the bench workload);
  - the per-feed path at Ns = 2048, the largest frame a step fills (Ns = 4096 needs 4097 samples: it never emits);
  - every channel scheduled with a "psd" source and both estimators at Ns = 4096 and I = 312 500 (100 ms), 8192 and
    4096 (one emission every other step, and every step).
Each step is timed on its own with CUDA events on the engine stream (after the inspector stream has been joined); the
mean step and the mean of the steps that emitted are reported.  A separate pass in the engine's timing mode gives the
device time of the "spectsrc_sched" family per step.  Card name and power limit first.

    python tools/spectsched_rate.py [--streams 296] [--steps 160]
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
    ap.add_argument("--steps", type=int, default=160)
    args = ap.parse_args()
    import torch
    import sigdigger_b200 as sdb
    import bench
    if sdb.device_count() < 1:
        raise SystemExit("spectsched_rate.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip())
    bench.FS, bench.N_FFT = 200e6, 65536
    S, N = args.streams, 65536
    n = 8 * N // 2
    base = torch.from_numpy(bench.make_base_signal("cfg3", n, seed=1)).cuda()
    x = base.unsqueeze(0).repeat(S, 1).contiguous()
    g = torch.Generator(device="cuda").manual_seed(1234)
    x += torch.view_as_complex(1e-3 * torch.randn((S, n, 2), generator=g, device="cuda"))
    torch.cuda.synchronize()

    def build(ns, I):
        e = sdb.Engine(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=n, samp_rate=bench.FS)
        hs = []
        for kind, f, baud, bw in bench.workload_channels("cfg3"):
            f0, bwa = bench.chan_angular(f, bw)
            h = e.open_channel(f0, bwa, 1.0)
            cls, kw = bench.insp_kwargs(kind, baud, e.channel_rate(h))
            e.set_inspector(h, cls, **kw)
            if ns:
                e.set_spectrum_source(h, "psd", ns)
                e.set_estimator(h, "baud-fac")
                e.set_estimator(h, "baud-nonlinear")
                if I:
                    e.set_spectrum_interval(h, I)
            hs.append(h)
        e.commit()
        return e, hs

    arms = [("off", 0, 0), ("per_feed", 2048, 0), ("sched", 4096, 312500), ("sched", 4096, 8192),
            ("sched", 4096, 4096)]
    for name, ns, I in arms:
        e, hs = build(ns, I)
        es = torch.cuda.ExternalStream(e.stream_ptr)

        def step():
            e.feed_device_ptr(x.data_ptr(), x.stride(0), n)

        for _ in range(4):
            step()
        e.sync()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        ev[0].record(es)
        emitted = []
        t = 4 * 4096 - 512                      # channel samples after the warm-up (the first hop primes the history)
        for k in range(args.steps):
            step()
            e.join()
            ev[k + 1].record(es)
            if I:
                emitted.append((t + 4096) // I > t // I and t + 4096 >= 4097)
            t += 4096
        e.sync()
        ms = [ev[k].elapsed_time(ev[k + 1]) for k in range(args.steps)]
        if I:
            n_last = len(e.read_spectra(hs[0])[1])
        e.timing(True)
        for _ in range(args.steps):
            step()
        e.sync()
        fam_ms, fam_n = e.kernel_time("spectsrc_sched")
        e.timing(False)
        em = [v for v, f in zip(ms, emitted) if f]
        row = dict(arm=name, ns=ns or None, interval=I or None, streams=S, steps=args.steps,
                   mean_step_ms=round(sum(ms) / len(ms), 4),
                   gsps=round(S * n / (sum(ms) / len(ms) * 1e-3) / 1e9, 2),
                   emitting_steps=len(em), emitting_step_ms=round(sum(em) / len(em), 4) if em else None,
                   quiet_step_ms=round(sum(v for v, f in zip(ms, emitted) if not f) / max(1, len(ms) - len(em)), 4)
                   if I else None,
                   spectsrc_sched_ms_per_launch_span=round(fam_ms, 4), spectsrc_sched_spans=fam_n,
                   last_step_emissions=n_last if I else None)
        print(json.dumps(row), flush=True)
        e.close()
        torch.cuda.synchronize()


if __name__ == "__main__":
    main()
