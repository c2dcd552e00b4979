"""FreeDV throughput on one GPU: 64 channels of gr_demod_freedv to the int16 modem stream and 64 channels of gr_mod_freedv from it
(make_gr_demod_freedv / make_gr_mod_freedv(125, 1e6, 1700, 2500, 200, MODE_1600, USB)), inputs resident in HBM.  Prints one JSON line
with, per block, the rate, per-stage device times, the HBM roofline of the bandwidth-bound stage, a full-size parity spot check
against the CPU oracle (tests/freedv_oracle.c) and the oracle's own rate on the host's threads as CPU baseline.

    python tools/freedv_bench.py [--no-cpu]

Reuses bench.py's helpers (data-sheet peak, CUDA-event timing, per-stage profile read-out, threaded CPU rate); writes nothing."""
import argparse
import ctypes as Ct
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import cpu_rate, host_cores, peaks, rx_stage_ms, timed_calls  # noqa: E402
from tests import freedv_oracle as FO  # noqa: E402


def freedv_rx_config_block(q, torch, dev, cores, cpu_seconds, C=64, T=1 << 22, k=3):
    """64 ch FreeDV RX up to the codec2 modem boundary (make_gr_demod_freedv(125,1e6,1700,2500,200,MODE_1600,USB)): /125 FIR (1045 taps)
    + complex side-band filter + agc2_ff + audio band-pass + int16 conversion, inputs resident in HBM.  Stage-1 roofline: 8 B read +
    8 / 125 B written per input sample = 8.064 B."""
    L = q.load_library()
    peak, _ = peaks()
    stream = torch.cuda.current_stream()
    torch.cuda.empty_cache()
    n_ = torch.arange(T, device=dev, dtype=torch.float64)
    f = 700.0 + 20.0 * torch.arange(C, device=dev, dtype=torch.float64)[:, None]
    X = (0.05 * torch.polar(torch.ones((C, T), device=dev, dtype=torch.float64), 2 * np.pi * f * n_ / 1e6)
         + 0.03 * torch.polar(torch.ones(T, device=dev, dtype=torch.float64), 2 * np.pi * 1900.0 * n_ / 1e6)).to(torch.complex64)
    X += torch.view_as_complex(torch.randn((C, T, 2), device=dev) * 0.01)
    blk = q.make_gr_demod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, n_channels=C, max_samples=T, device=dev.index)
    blk.set_stream(stream.cuda_stream)
    blk.work_device(X.data_ptr(), T, T)
    torch.cuda.synchronize()
    got0, got1 = blk.read_port(0), blk.read_port(1)
    chans = [0, C // 2, C - 1]
    ident, items = True, 0
    for c in chans:
        w0, w1 = FO.FreedvRx(125, 1000000, 2500, 200, 0).work(X[c].cpu().numpy())
        ident = ident and np.array_equal(got0[c], w0) and np.array_equal(got1[c], w1) and len(w1) == len(w0) == (T + 124) // 125
        items += len(w0) + len(w1)
    del got0, got1
    L.qrl_rx_profile(blk._h, 1)
    ms = timed_calls(lambda: blk.work_device(X.data_ptr(), T, T), k, stream, torch, warm=1)
    st = rx_stage_ms(L, blk)
    L.qrl_rx_profile(blk._h, 0)
    fir_ms, fir_n = st["stage1_fir"]
    fir_avg = fir_ms / max(1, fir_n)
    per_call = max(1, fir_n // (k + 1))
    alg = 8.064 * C * T / per_call
    res = {"workload": "64ch FreeDV RX to the int16 modem stream (make_gr_demod_freedv(125,1e6,1700,2500,200,MODE_1600,0)), T=2^22 per call",
           "channels": C, "samples_per_channel_per_call": T, "ms_per_call": ms, "value": C * T / ms / 1e3, "unit": "Msamples/s",
           "realtime_factor_per_channel": T / ms / 1e3,
           "stage_ms_per_call": {"stage1_fir": st["stage1_fir"][0] / (k + 1), "sideband_filter": st["chan_filter"][0] / (k + 1),
                                 "agc_audio_int16": st["symbol_sync_or_audio"][0] / (k + 1)},
           "roofline": {"kernel": "fir_decim_poly_kernel<125,9,8,48,6>", "bound": "hbm", "achieved": alg / (fir_avg * 1e-3) / 1e9 if fir_avg > 0 else 0.0,
                        "peak": peak, "unit": "GB/s", "frac": (alg / (fir_avg * 1e-3) / 1e9 / peak) if fir_avg > 0 else 0.0,
                        "algorithmic_bytes_per_launch": alg, "avg_launch_ms": fir_avg, "launches_per_call": per_call,
                        "whole_chain_frac": 8.064 * C * T / (ms * 1e-3) / 1e9 / peak},
           "parity_vs_oracle": {"channels": chans, "ports_bit_identical": bool(ident), "items_compared": int(items)}}
    if cpu_seconds > 0:
        xs = [X[c % C, : 1 << 20].cpu().numpy().copy() for c in range(min(cores, 8))]

        def mk(i):
            r = FO.FreedvRx(125, 1000000, 2500, 200, 0)
            x = xs[i % len(xs)]
            return lambda: r.work(x)
        v, dt = cpu_rate(mk, cores, cpu_seconds, 1 << 20)
        res["cpu_baseline"] = {"value": v, "unit": "Msamples/s", "cores": cores, "kind": "port",
                               "sample": "%d host threads x 2^20-sample chunks of the same chain (CPU oracle port) for %.1f s" % (cores, dt)}
        res["gpu_over_cpu"] = res["value"] / v if v > 0 else None
    blk.close()
    del X
    return res


def freedv_tx_config_block(q, torch, dev, cores, cpu_seconds, C=64, n=32768, k=10):
    """64 ch FreeDV TX behind the codec2 modem (make_gr_mod_freedv(125,1e6,1700,2500,200,MODE_1600,USB)): int16 -> side-band filter ->
    feedforward AGC (512) -> x125 interpolating FIR (2007 taps) x0.98 x bb_gain.  Interpolator roofline: 8 B written per output sample."""
    L = q.load_library()
    peak, _ = peaks()
    stream = torch.cuda.current_stream()
    torch.cuda.empty_cache()
    rng = np.random.default_rng(5100)
    t = np.arange(n) / 8000.0
    data_h = np.stack([(6000 * np.sin(2 * np.pi * (600 + 15 * c) * t) + 4000 * np.sin(2 * np.pi * 1700 * t)
                        + 500 * rng.standard_normal(n)).astype(np.int16) for c in range(C)])
    data = torch.from_numpy(data_h).to(dev)
    tx = q.make_gr_mod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, n_channels=C, max_items=n, device=dev.index)
    tx.set_stream(stream.cuda_stream)
    nout = 125 * n
    tx.work_device(data.data_ptr(), n, n); tx.sync()
    out = torch.empty((C, nout), dtype=torch.complex64, device=dev)
    n2 = Ct.c_long()
    assert L.qrl_tx_read(tx._h, Ct.c_void_p(out.data_ptr()), nout, Ct.byref(n2), 1) == 0 and n2.value == nout
    chans = [0, C // 2, C - 1]
    ident = True
    for c in chans:
        w = FO.FreedvTx(125, 1000000, 2500, 200, 0).work(data_h[c])
        g = out[c].cpu().numpy()
        ident = ident and len(w) == len(g) and np.array_equal(w.view(np.float32), g.view(np.float32))
    del out
    L.qrl_tx_profile(tx._h, 1)
    ms = timed_calls(lambda: tx.work_device(data.data_ptr(), n, n), k, stream, torch, warm=1)
    st = {}
    for s_, nm in enumerate(("int16_sideband_filter", "feedforward_agc", "interp_fir")):
        mm, cc = Ct.c_double(), Ct.c_long()
        L.qrl_tx_profile_read(tx._h, s_, Ct.byref(mm), Ct.byref(cc))
        st[nm] = mm.value / (k + 1)
        if s_ == 2:
            interp_avg = mm.value / max(1, cc.value)
    L.qrl_tx_profile(tx._h, 0)
    alg = 8.0 * C * nout
    res = {"workload": "64ch FreeDV TX from the int16 modem stream (make_gr_mod_freedv(125,1e6,1700,2500,200,MODE_1600,0)), 32768 modem samples per call",
           "channels": C, "modem_samples_per_channel_per_call": n, "out_samples_per_channel_per_call": nout, "ms_per_call": ms,
           "value": C * nout / ms / 1e3, "unit": "Msamples/s (output)", "stage_ms_per_call": st,
           "roofline": {"kernel": "interp_fir_ccf_rt_kernel<125,17,8,4>", "bound": "hbm", "achieved": alg / (interp_avg * 1e-3) / 1e9 if interp_avg > 0 else 0.0,
                        "peak": peak, "unit": "GB/s", "frac": (alg / (interp_avg * 1e-3) / 1e9 / peak) if interp_avg > 0 else 0.0,
                        "algorithmic_bytes_per_launch": alg, "avg_launch_ms": interp_avg, "launches_per_call": 1,
                        "whole_chain_frac": alg / (ms * 1e-3) / 1e9 / peak},
           "parity_vs_oracle": {"channels": chans, "iq_bit_identical": bool(ident), "samples_compared": 3 * nout}}
    if cpu_seconds > 0:
        def mk(i):
            o = FO.FreedvTx(125, 1000000, 2500, 200, 0)
            d = data_h[i % C][:1024]
            return lambda: o.work(d)
        v, dt = cpu_rate(mk, cores, cpu_seconds, 1024 * 125)
        res["cpu_baseline"] = {"value": v, "unit": "Msamples/s (output)", "cores": cores, "kind": "port",
                               "sample": "%d host threads x 1024-sample modem bursts through the oracle's FreeDV modulator for %.1f s" % (cores, dt)}
        res["gpu_over_cpu"] = res["value"] / v if v > 0 else None
    tx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-cpu", action="store_true", help="skip the CPU baselines")
    args = ap.parse_args()
    import torch
    import qradiolink_b200 as q
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cores, _ = host_cores()
    cs = 0.0 if args.no_cpu else 4.0
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    # the handles run on a real torch stream (a NULL stream handle would give them their own, which the timing events do not see)
    with torch.cuda.stream(torch.cuda.Stream(dev)):
        out = {"gpu": gpu, "freedv_rx_64ch": freedv_rx_config_block(q, torch, dev, cores, cs),
               "freedv_tx_64ch": freedv_tx_config_block(q, torch, dev, cores, cs)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
