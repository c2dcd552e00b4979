"""Transmit front-end throughput on one GPU: 64 channels of qrl_tx_frontend (gr_mod_base's carrier-offset rotator at 1 Msps + x N
interpolator, about 210 taps per arm) at 2, 10 and 20 Msps, inputs resident in HBM.  Prints one JSON line with, per rate, ms per call,
output Gsamples/s, the interpolating kernel's FP32 issue fraction (2 NT FFMA per output over the kernel's own time from torch.profiler,
against SMs x 128 FFMA per clock at the card's maximum SM clock), a full-size parity spot check of three channels against the CPU oracle
(tests/tx_frontend_oracle.c) and the oracle's own rate on the host's threads; and the card, its power limit and SM clocks.

    python tools/tx_frontend_bench.py [--no-cpu] [--n 65536]

Reuses bench.py's helpers (CUDA-event timing, threaded CPU rate); writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import cpu_rate, host_cores, timed_calls  # noqa: E402
from tests import tx_frontend_oracle as TO  # noqa: E402


def _kernel_ms(torch, fn, k, name):
    """device time per call of the kernels whose name contains `name`, from a torch.profiler trace of k calls"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(k):
            fn()
        torch.cuda.synchronize()
    us = 0.0
    for e in prof.key_averages():
        if name in e.key:
            us += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
    return us / 1e3 / k


def rate_block(q, torch, dev, samp_rate, cores, cpu_seconds, sm_count, sm_clock_mhz, C=64, n=1 << 16, k=10):
    N = samp_rate // 1000000
    stream = torch.cuda.current_stream()
    torch.cuda.empty_cache()
    t = torch.arange(n, device=dev, dtype=torch.float64)
    f = -200000.0 + 6000.0 * torch.arange(C, device=dev, dtype=torch.float64)[:, None]
    X = (0.4 * torch.polar(torch.ones((C, n), device=dev, dtype=torch.float64), 2 * np.pi * f * t / 1e6)).to(torch.complex64)
    X += torch.view_as_complex(torch.randn((C, n, 2), device=dev) * 0.05)
    fe = q.TxFrontend(samp_rate, n_channels=C, max_in=n, device=dev.index)
    fe.set_stream(stream.cuda_stream)
    offsets = [-150000.0 + 5000.0 * c for c in range(C)]
    for c, hz in enumerate(offsets):
        fe.set_carrier_offset(hz, channel=c)
    # parity: the first call, against fresh oracles
    assert fe.work_device(X.data_ptr(), n, n) == N * n
    got = fe.read()
    chans = [0, C // 2, C - 1]
    ident = True
    for c in chans:
        o = TO.TxFrontend(samp_rate); o.set_carrier_offset(offsets[c])
        w = o.work(X[c].cpu().numpy())
        ident = ident and len(w) == got.shape[1] and np.array_equal(w.view(np.uint32), got[c].view(np.uint32))
    del got
    call = lambda: fe.work_device(X.data_ptr(), n, n)                     # noqa: E731
    ms = timed_calls(call, k, stream, torch, warm=2)
    kern_ms = _kernel_ms(torch, call, k, "tx_frontend_interp_kernel") if N >= 2 else 0.0
    ntaps = TO.TxFrontend(samp_rate).ntaps
    nt = (ntaps + N - 1) // N
    outs = C * n * N
    ffma = 2.0 * nt * outs
    peak_ffma = sm_count * 128 * sm_clock_mhz * 1e6
    res = {"samp_rate": samp_rate, "interpolation": N, "ntaps": ntaps, "taps_per_arm": nt, "channels": C, "in_samples_per_channel_per_call": n,
           "ms_per_call": ms, "out_gsamples_per_s": outs / (ms * 1e-3) / 1e9,
           "interp_kernel": {"kernel": "tx_frontend_interp_kernel<10,18>", "bound": "fp32 issue", "ms_per_call": kern_ms,
                             "algorithmic_ffma_per_call": ffma,
                             "achieved_tffma_per_s": ffma / (kern_ms * 1e-3) / 1e12 if kern_ms > 0 else 0.0,
                             "peak_tffma_per_s": peak_ffma / 1e12,
                             "frac": ffma / (kern_ms * 1e-3) / peak_ffma if kern_ms > 0 else 0.0,
                             "peak_basis": "%d SMs x 128 FFMA/clk x %d MHz (max SM clock)" % (sm_count, sm_clock_mhz)},
           "realtime_factor_per_channel": n / (ms * 1e-3) / 1e6,
           "parity_vs_oracle": {"channels": chans, "iq_bit_identical": bool(ident), "samples_compared": 3 * N * n}}
    if cpu_seconds > 0:
        xs = [X[c % C, :4096].cpu().numpy().copy() for c in range(min(cores, 8))]

        def mk(i):
            o = TO.TxFrontend(samp_rate); o.set_carrier_offset(offsets[i % C])
            x = xs[i % len(xs)]
            return lambda: o.work(x)
        v, dt = cpu_rate(mk, cores, cpu_seconds, 4096 * N)
        res["cpu_baseline"] = {"value": v / 1e3, "unit": "Gsamples/s (output)", "cores": cores, "kind": "oracle",
                               "sample": "%d host threads x 4096-sample chunks through the oracle's front end for %.1f s" % (cores, dt)}
        res["gpu_over_cpu"] = res["out_gsamples_per_s"] / (v / 1e3) if v > 0 else None
    fe.close()
    del X
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-cpu", action="store_true", help="skip the CPU baselines")
    ap.add_argument("--n", type=int, default=1 << 16, help="input samples per channel per call (1 Msps)")
    args = ap.parse_args()
    import torch
    import qradiolink_b200 as q
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cores, _ = host_cores()
    cs = 0.0 if args.no_cpu else 3.0
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip()
    fields = [s.strip() for s in smi.split(",")]
    name, power, sm_max, sm_now = (fields + ["?"] * 4)[:4]
    sm_count = torch.cuda.get_device_properties(dev).multi_processor_count
    try:
        clk = int(float(sm_max))
    except ValueError:
        clk = 1980
    out = {"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": sm_max, "sm_clock_at_start_mhz": sm_now, "sm_count": sm_count}
    # the handle runs on a real torch stream (a NULL stream handle would give it its own, which the timing events do not see)
    with torch.cuda.stream(torch.cuda.Stream(dev)):
        for fs in (2000000, 10000000, 20000000):
            out["tx_frontend_64ch_%dmsps" % (fs // 1000000)] = rate_block(q, torch, dev, fs, cores, cs, sm_count, clk, n=args.n)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
