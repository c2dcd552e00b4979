"""Receive front-end throughput on one GPU for one wideband stream feeding every channel (qrl_frontend_work with stride 0: one SDR,
C receivers at C carrier offsets).  Workloads: 64 channels at 2, 10, 20, 32 and 33 Msps (32 is the top of frontend_shared_kernel's
range, 33 runs frontend_fir_kernel on the one stream) and 256 channels at 10 Msps, one capture resident in HBM, each call's input
larger than the L2.  Prints one JSON line with, per workload:
  * the shared path: ms per call, wideband Msamples/s in, channel Msamples/s out, the real-time factor per channel;
  * the FIR kernel's share of FP32 FFMA issue: 2 ntaps FFMA per output per channel over the kernel's own time (torch.profiler),
    against SMs x 128 FFMA per clock at the SM clock sampled while calls are running;
  * the same call through the per-channel path fed a [C][T] slab of C identical rows (what a caller without stride 0 does), timed in
    the same process, alternating with the shared path;
  * a full-size parity check of three channels against the CPU oracle;
and one host-fed run (pinned memory, 64 channels at 10 Msps), with the card, its power limit and SM clocks.

    python tools/frontend_bench.py [--T 8388608] [--rounds 5]

Reuses bench.py's CUDA-event timing; writes nothing."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import timed_calls  # noqa: E402

TOP_TILED = 32


def _smi(fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader,nounits"], capture_output=True,
                         text=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


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


def _sm_clock_under_load(torch, fn, k):
    """SM clock (MHz) read while k calls are queued on the GPU"""
    for _ in range(k):
        fn()
    mhz = _smi("clocks.sm")[0]
    torch.cuda.synchronize()
    try:
        return float(mhz)
    except ValueError:
        return None


def workload(q, oracle, torch, dev, samp_rate, Cn, T, rounds, k, sm_count):
    D = samp_rate // 1000000
    torch.cuda.empty_cache()
    t = torch.arange(T, device=dev, dtype=torch.float64)
    X = torch.zeros(T, device=dev, dtype=torch.complex64)
    for f in (-0.41, -0.17, 0.05, 0.29, 0.44):
        X += (0.15 * torch.polar(torch.ones_like(t), 2 * np.pi * f * t)).to(torch.complex64)
    X += torch.view_as_complex(torch.randn((T, 2), device=dev) * 0.05)
    del t
    offsets = [(-0.45 + 0.9 * c / Cn) * samp_rate for c in range(Cn)]
    stream = torch.cuda.current_stream()
    fe = q.Frontend(samp_rate, n_channels=Cn, max_in=T, device=dev.index)
    fe.set_stream(stream.cuda_stream)
    for c, hz in enumerate(offsets):
        fe.set_carrier_offset(hz, channel=c)
    # parity: the first call, against fresh oracles
    nout = fe.work_device(X.data_ptr(), T, 0)
    out = np.zeros((Cn, nout), np.complex64)
    assert q.load_library().qrl_frontend_read(fe._h, out.ctypes.data_as(C.c_void_p), nout) == 0
    xh = X.cpu().numpy()
    chans = [0, Cn // 2, Cn - 1]
    ident = True
    for c in chans:
        o = oracle.Frontend(samp_rate); o.set_carrier_offset(offsets[c])
        w = o.work(xh)
        ident = ident and len(w) == nout and np.array_equal(w.view(np.uint32), out[c].view(np.uint32))
    ntaps = oracle.Frontend(samp_rate).ntaps
    del out, xh
    # the per-channel path on C identical rows
    slab = X[None, :].expand(Cn, T).contiguous()
    fe_rows = q.Frontend(samp_rate, n_channels=Cn, max_in=T, device=dev.index)
    fe_rows.set_stream(stream.cuda_stream)
    for c, hz in enumerate(offsets):
        fe_rows.set_carrier_offset(hz, channel=c)
    shared = lambda: fe.work_device(X.data_ptr(), T, 0)              # noqa: E731
    rows = lambda: fe_rows.work_device(slab.data_ptr(), T, T)        # noqa: E731
    ms_s, ms_r = [], []
    for _ in range(rounds):
        ms_s.append(timed_calls(shared, k, stream, torch, warm=1))
        ms_r.append(timed_calls(rows, k, stream, torch, warm=1))
    kname = "frontend_shared_kernel" if D <= TOP_TILED else "frontend_fir_kernel"
    kern_ms = _kernel_ms(torch, shared, k, kname)
    mhz = _sm_clock_under_load(torch, shared, max(k, 20))
    ms, ms_rows = float(np.median(ms_s)), float(np.median(ms_r))
    outs = Cn * (T // D)
    ffma = 2.0 * ntaps * outs
    peak = sm_count * 128 * (mhz or 0) * 1e6
    res = {"samp_rate": samp_rate, "decimation": D, "ntaps": ntaps, "channels": Cn, "wideband_samples_per_call": T,
           "shared": {"ms_per_call": ms, "ms_per_call_rounds": ms_s, "wideband_msamples_per_s": T / (ms * 1e-3) / 1e6,
                      "channel_msamples_per_s_out": outs / (ms * 1e-3) / 1e6, "realtime_factor_per_channel": T / D / (ms * 1e-3) / 1e6},
           "fir_kernel": {"kernel": kname, "bound": "fp32 issue", "ms_per_call": kern_ms, "fir_ffma_per_call": ffma,
                          "sm_clock_sampled_mhz": mhz, "peak_basis": "%d SMs x 128 FFMA/clk x sampled SM clock" % sm_count,
                          "fp32_issue_frac": ffma / (kern_ms * 1e-3) / peak if kern_ms > 0 and peak > 0 else None},
           "replicated_rows": {"ms_per_call": ms_rows, "ms_per_call_rounds": ms_r, "channel_msamples_per_s_out": outs / (ms_rows * 1e-3) / 1e6},
           "shared_speedup_over_rows": ms_rows / ms,
           "parity_vs_oracle": {"channels": chans, "iq_bit_identical": bool(ident), "samples_compared": 3 * nout}}
    fe.close(); fe_rows.close()
    del slab, X
    return res


def host_fed(q, torch, dev, samp_rate, Cn, T, k):
    """wideband stream from pinned host memory: copy T samples once per call, output stays in HBM"""
    D = samp_rate // 1000000
    stream = torch.cuda.current_stream()
    xh = torch.view_as_complex(torch.randn((T, 2)) * 0.3).pin_memory()
    fe = q.Frontend(samp_rate, n_channels=Cn, max_in=T, device=dev.index)
    fe.set_stream(stream.cuda_stream)
    for c in range(Cn):
        fe.set_carrier_offset((-0.45 + 0.9 * c / Cn) * samp_rate, channel=c)
    L = q.load_library()
    n = C.c_long()
    call = lambda: L.qrl_frontend_work(fe._h, C.c_void_p(xh.data_ptr()), T, 0, 0, C.byref(n))    # noqa: E731
    ms = timed_calls(call, k, stream, torch, warm=2)
    fe.close()
    return {"samp_rate": samp_rate, "channels": Cn, "wideband_samples_per_call": T, "ms_per_call": ms,
            "wideband_msamples_per_s": T / (ms * 1e-3) / 1e6, "channel_msamples_per_s_out": Cn * (T // D) / (ms * 1e-3) / 1e6,
            "input": "pinned host memory, one H2D copy of T samples per call"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=1 << 23, help="wideband samples per call (8 B each; default 64 MiB, above the L2)")
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of the shared and the replicated-rows path")
    ap.add_argument("--k", type=int, default=5, help="calls per timed round")
    args = ap.parse_args()
    import torch
    import qradiolink_b200 as q
    from oracle import oracle as O
    O.lib()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power, sm_max, sm_now = (_smi("name,power.limit,clocks.max.sm,clocks.sm") + ["?"] * 4)[:4]
    sm_count = torch.cuda.get_device_properties(dev).multi_processor_count
    out = {"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": sm_max, "sm_clock_at_start_mhz": sm_now, "sm_count": sm_count}
    # the handles run on a real torch stream (a NULL stream handle would give each its own, which the timing events do not see)
    with torch.cuda.stream(torch.cuda.Stream(dev)):
        for fs, Cn in ((2000000, 64), (10000000, 64), (20000000, 64), (TOP_TILED * 1000000, 64), ((TOP_TILED + 1) * 1000000, 64),
                       (10000000, 256)):
            out["shared_%dch_%dmsps" % (Cn, fs // 1000000)] = workload(q, O, torch, dev, fs, Cn, args.T, args.rounds, args.k, sm_count)
        out["host_fed_64ch_10msps"] = host_fed(q, torch, dev, 10000000, 64, args.T, args.k)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
