"""Throughput of the DMR direct-mode (DMO) burst decoder (qrl_dmr_dmo_rx: dmr_dmo_sink_kernel + dmr_decode_kernel) on the GPU.

4096 channels x 2^16 port-3 samples per call (2.7 s of 24 ksps per channel), input already in HBM, CUDA events around the calls after
warm-up.  Two workloads, reported separately:
  * locked: every channel receives back-to-back MS voice superframes (one burst per 1440 samples);
  * search: every channel receives Gaussian noise, which passes the 24-symbol sign prefilter now and then, so the sink stays searching.
Per workload: ms per call, Msamples/s, bursts/s, the fraction of the H100's data-sheet HBM rate (4 bytes per input sample over
3.35 TB/s), and the compiled reference's gr_dmr_dmo_sink on one host core (oracle/_ref/libqrl_ref_dmr_dmo.so, if built) in the same run.

    python tools/dmr_dmo_bench.py [--channels 4096] [--samples 65536] [--steps 20] [--warmup 3]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def voice_period(rng):
    from tests import dmr_dmo_model as D
    return D.to_samples(D.voice_superframe(rng, cc=1), rng=rng, noise=0.02)        # 8640 samples: 6 bursts


def ref_rate(x):
    path = os.path.join(ROOT, "oracle", "_ref", "libqrl_ref_dmr_dmo.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.ref_dmo_create.restype = C.c_void_p
    h = C.c_void_p(L.ref_dmo_create())
    out = np.zeros((len(x) // 270 + 2, 72), np.uint8)
    x = np.ascontiguousarray(x, np.float32)
    t = time.perf_counter()
    L.ref_dmo_work(h, x.ctypes.data_as(C.c_void_p), C.c_long(len(x)), 0, out.ctypes.data_as(C.c_void_p), len(out))
    dt = time.perf_counter() - t
    L.ref_dmo_destroy(h)
    return len(x) / dt / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=4096)
    ap.add_argument("--samples", type=int, default=1 << 16)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    import qradiolink_b200 as q
    if q.device_count() < 1:
        raise SystemExit("dmr_dmo_bench needs a CUDA device")
    Cn, N = a.channels, a.samples
    rng = np.random.default_rng(1)
    period = voice_period(rng)
    P = len(period)
    stride = N + P
    dev = torch.device("cuda:0")
    results = []
    for name in ("locked", "search"):
        if name == "locked":
            row = np.tile(period, stride // P + 2)
            base = torch.from_numpy(row).to(dev)
            # channel c starts 37 c samples into the period; call k reads at offset (k N) mod P, so the stream is continuous
            idx = (torch.arange(stride, device=dev, dtype=torch.int32)[None, :] + 37 * torch.arange(Cn, device=dev, dtype=torch.int32)[:, None]) % P
            buf = base[idx].contiguous()
        else:
            g = torch.Generator(device=dev).manual_seed(7)
            buf = torch.randn((Cn, stride), generator=g, device=dev, dtype=torch.float32) * 0.5
            P = 0
        dec = q.DmrDmoBurstDecoder(Cn, N, ambe_fec=True)
        stream = torch.cuda.Stream()
        dec.set_stream(stream.cuda_stream)     # the events below and the calls share one stream
        torch.cuda.synchronize()

        def call(k):
            off = (k * N) % P if P else 0
            dec.work_device(buf.data_ptr() + 4 * off, N, stride)

        for k in range(a.warmup):
            call(k)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for k in range(a.warmup, a.warmup + a.steps):
            call(k)
        e1.record(stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / a.steps
        per_call_bursts = sum(len(r) for r in dec.read())
        samples = Cn * N
        ref = ref_rate(np.tile(period, (1 << 20) // len(period) + 1) if name == "locked" else
                       (np.random.default_rng(7).standard_normal(1 << 20) * 0.5).astype(np.float32))
        res = {"workload": name, "channels": Cn, "samples_per_call": N, "ms_per_call": round(ms, 4),
               "msamples_per_s": round(samples / ms / 1e3, 1), "bursts_per_s": round(per_call_bursts / ms * 1e3, 1),
               "bursts_last_call": per_call_bursts, "hbm_fraction": round(samples * 4 / (ms * 1e-3) / HBM_BYTES_PER_S, 4),
               "ref_one_core_msamples_per_s": None if ref is None else round(ref, 2),
               "gpu": torch.cuda.get_device_name(0)}
        print(json.dumps(res))
        results.append(res)
        dec.close()
        del buf
        torch.cuda.empty_cache()
    return results


if __name__ == "__main__":
    main()
