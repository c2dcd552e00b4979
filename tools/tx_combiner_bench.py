"""Transmit combiner throughput on one GPU: qrl_tx_combiner (per channel gr_mod_base's x N interpolator, about 210 taps per arm, a rotator
at the device rate, the channel sum, x 1 / C, x bb_gain into ONE stream) for 64 channels at 2 / 10 / 20 Msps and 256 channels at 10 Msps,
n = 65 536 inputs per channel resident in HBM.  Prints one JSON line with the card, its power limit and the SM clock sampled after each
case and, per case:
  * ms per call, wideband Msamples/s out, real-time factor per channel;
  * tx_combiner_kernel's FP32 issue fraction: C 2 NT FFMA per wideband output over the kernel's own time from torch.profiler, against
    SMs x 128 FFMA per clock at the card's maximum SM clock;
  * the composed path a user has without the combiner, timed alternately in the same run: qrl_tx_frontend at offset 0 ([C][N n] to
    HBM), then a torch rotate-and-sum against a precomputed phasor table (its time excludes building the table);
  * the first call's first P input samples per channel compared bit for bit with the CPU oracle (tests/tx_combiner_oracle.c).

    python tools/tx_combiner_bench.py [--n 65536] [--k 10]

Reuses bench.py's CUDA-event timing; writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import timed_calls  # noqa: E402
from tests import tx_combiner_oracle as TCO  # noqa: E402


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


def _smi(fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return [s.strip() for s in out.stdout.strip().split(",")]


class _DevRows:
    """zero-copy torch view of a library buffer (device pointer, [rows][cols] complex64 with a row stride)"""

    def __init__(self, ptr, rows, cols, stride):
        self.__cuda_array_interface__ = {"shape": (rows, cols), "strides": (8 * stride, 8), "typestr": "<c8", "data": (ptr, False),
                                         "version": 2}


def case(q, torch, dev, samp_rate, C, n, k, sm_count, clk, prefix):
    N = samp_rate // 1000000
    stream = torch.cuda.current_stream()
    torch.cuda.empty_cache()
    t = torch.arange(n, device=dev, dtype=torch.float64)
    f = -200000.0 + 6000.0 * (torch.arange(C, device=dev, dtype=torch.float64)[:, None] % 64)
    X = (0.4 * torch.polar(torch.ones((C, n), device=dev, dtype=torch.float64), 2 * np.pi * f * t / 1e6)).to(torch.complex64)
    X += torch.view_as_complex(torch.randn((C, n, 2), device=dev) * 0.05)
    rows = [X[c].data_ptr() for c in range(C)]
    half = samp_rate / 2 - 500000.0
    offsets = [-half + 2 * half * c / (C - 1) for c in range(C)]
    comb = q.TxCombiner(samp_rate, n_channels=C, max_in=n, device=dev.index)
    comb.set_stream(stream.cuda_stream)
    for c, hz in enumerate(offsets):
        comb.set_carrier_offset(hz, channel=c)
    assert comb.work_device(rows, n) == N * n
    got = comb.read()[:N * prefix]
    o = TCO.TxCombiner(samp_rate, C)
    for c, hz in enumerate(offsets):
        o.set_carrier_offset(hz, c)
    want = o.work(X[:, :prefix].cpu().numpy())
    ident = bool(np.array_equal(got.view(np.uint32), want.view(np.uint32)))
    del got

    # the composed path: per-channel device-rate streams to HBM, then rotate and sum in torch
    fe = q.TxFrontend(samp_rate, n_channels=C, max_in=n, device=dev.index)
    fe.set_stream(stream.cuda_stream)
    fe.work_device(X.data_ptr(), n, n)
    p, st, m = fe.out_device()
    U = torch.as_tensor(_DevRows(p, C, m, st), device=dev)
    nn = torch.arange(N * n, device=dev, dtype=torch.float64)
    inc = torch.tensor([np.rint(hz / samp_rate * 2 ** 32) / 2 ** 32 for hz in offsets], device=dev, dtype=torch.float64)[:, None]
    rot = torch.polar(torch.ones((C, N * n), device=dev, dtype=torch.float64), 2 * np.pi * ((inc * nn) % 1.0)).to(torch.complex64)
    y = torch.empty(N * n, device=dev, dtype=torch.complex64)

    def composed():
        fe.work_device(X.data_ptr(), n, n)
        torch.mul(torch.sum(U * rot, 0), 1.0 / C, out=y)

    fused = lambda: comb.work_device(rows, n)                              # noqa: E731
    ms_f, ms_c = [], []
    for _ in range(3):                                                     # alternated, so both see the same clocks and neighbours
        ms_f.append(timed_calls(fused, k, stream, torch, warm=2))
        ms_c.append(timed_calls(composed, k, stream, torch, warm=1))
    sm_clock = _smi("clocks.sm")[0]
    ms, msc = float(np.median(ms_f)), float(np.median(ms_c))
    kern_ms = _kernel_ms(torch, fused, k, "tx_combiner_kernel") if N >= 2 else 0.0
    nt = (o.ntaps + N - 1) // N
    outs = N * n
    ffma = float(C) * 2.0 * nt * outs
    peak = sm_count * 128 * clk * 1e6
    res = {"samp_rate": samp_rate, "interpolation": N, "channels": C, "in_samples_per_channel_per_call": n, "taps_per_arm": nt,
           "ms_per_call": ms, "ms_per_call_runs": ms_f, "wideband_msamples_per_s": outs / (ms * 1e-3) / 1e6,
           "realtime_factor_per_channel": n / (ms * 1e-3) / 1e6,
           "kernel": {"name": "tx_combiner_kernel<10,18>", "bound": "fp32 issue", "ms_per_call": kern_ms, "algorithmic_ffma_per_call": ffma,
                      "frac": ffma / (kern_ms * 1e-3) / peak if kern_ms > 0 else 0.0,
                      "peak_basis": "%d SMs x 128 FFMA/clk x %d MHz (max SM clock)" % (sm_count, clk)},
           "composed_path": {"what": "qrl_tx_frontend at offset 0, then torch (U * phasors).sum(0) / C", "ms_per_call": msc,
                             "ms_per_call_runs": ms_c, "fused_speedup": msc / ms},
           "sm_clock_sampled_mhz": sm_clock,
           "parity_vs_oracle": {"first_call_prefix_inputs_per_channel": prefix, "iq_bit_identical": ident, "samples_compared": N * prefix}}
    comb.close(); fe.close()
    del X, U, rot, y
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 16, help="input samples per channel per call (1 Msps)")
    ap.add_argument("--k", type=int, default=10, help="timed calls per run")
    ap.add_argument("--prefix", type=int, default=2048, help="input samples per channel compared with the oracle")
    args = ap.parse_args()
    import torch
    import qradiolink_b200 as q
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power, sm_max, sm_now = (_smi("name,power.limit,clocks.max.sm,clocks.sm") + ["?"] * 4)[:4]
    sm_count = torch.cuda.get_device_properties(dev).multi_processor_count
    try:
        clk = int(float(sm_max))
    except ValueError:
        clk = 1980
    out = {"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": sm_max, "sm_clock_at_start_mhz": sm_now, "sm_count": sm_count}
    # the handles run on a real torch stream (a NULL stream handle would give them their own, which the timing events do not see)
    with torch.cuda.stream(torch.cuda.Stream(dev)):
        for fs, C in ((2000000, 64), (10000000, 64), (20000000, 64), (10000000, 256)):
            out["tx_combiner_%dch_%dmsps" % (C, fs // 1000000)] = case(q, torch, dev, fs, C, args.n, args.k, sm_count, clk, args.prefix)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
