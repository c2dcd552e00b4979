"""Polyphase channelizer / synthesizer throughput on one GPU (qrl_pfb_*), 2^24 wideband samples per call resident in HBM.

Shapes (M channels at wideband rate fs; prototypes qrl_firdes_low_pass_2(1, fs, 5000, 2000, 60, Blackman-Harris), the reference's
MMDVM design scaled to fs, gain M for the synthesizer):
  * M <= 64: (10, 250 kHz), the register-tiled reference shape; (64, 1.6 MHz); tests/test_gpu_pfb.py's GENERIC_SHAPES (33, 1000 taps)
    and (64, 8192 taps) with random taps at 1.6 MHz;
  * the 25 kHz grid: (256, 6.4 MHz), (400, 10 MHz), (1024, 25.6 MHz), (4096, 102.4 MHz).
For each shape and direction: ms per call, wideband Gsamples/s, x real time at fs, FFMA per wideband sample (4 M + 2 tpf), and for
the two-kernel shapes each kernel's time from torch.profiler with pfb_dft_kernel's and the whole call's share of FP32 FFMA issue
(SMs x 128 FFMA per clock at the SM clock sampled under load in the same run).  `--lib PATH` times another build of libqrl_b200.so
(e.g. the parent commit's) on the same shapes, alternating with this one; its outputs are compared bit for bit with this build's.
End to end, the MMDVM bank: 10 Msps -> channelizer M = 400 -> qrl_mmdvm_rx over all 400 rows, ms per call and x real time.

    python tools/pfb_bench.py [--k 5] [--lib OTHER/libqrl_b200.so] [--only M,M,..]

Prints one JSON line; writes nothing."""
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

N_WIDE = 1 << 24
CHANNELIZER, SYNTHESIZER = 201, 202
# (label, M, fs, ntaps or None for the low_pass_2 prototype)
SHAPES = [("m10_250k", 10, 250e3, None), ("m64_1m6", 64, 1.6e6, None), ("m33_1000taps", 33, 1.6e6, 1000),
          ("m64_8192taps", 64, 1.6e6, 8192), ("m256_6m4", 256, 6.4e6, None), ("m400_10m", 400, 10e6, None),
          ("m1024_25m6", 1024, 25.6e6, None), ("m4096_102m4", 4096, 102.4e6, None)]


def _smi(fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return [s.strip() for s in out.stdout.strip().split(",")]


def _open(path):
    from qradiolink_b200.lib import SYMBOLS
    L = C.CDLL(path)
    for name in ("qrl_pfb_create", "qrl_pfb_destroy", "qrl_pfb_set_stream", "qrl_pfb_work", "qrl_pfb_out_device", "qrl_last_error",
                 "qrl_firdes_low_pass_2"):
        fn = getattr(L, name)
        fn.restype, fn.argtypes = SYMBOLS[name]
    return L


class Pfb:
    """one qrl_pfb handle of library L, driven with device input on `stream`"""

    def __init__(self, L, kind, M, taps, max_in, stream):
        self.L, self.kind, self.M = L, kind, M
        self.h = C.c_void_p()
        t = np.ascontiguousarray(taps, np.float32)
        rc = L.qrl_pfb_create(kind, M, t.ctypes.data_as(C.c_void_p), len(t), max_in, 0, C.byref(self.h))
        if rc:
            raise RuntimeError("qrl_pfb_create(%d, %d) failed: %s" % (kind, M, L.qrl_last_error(None)))
        L.qrl_pfb_set_stream(self.h, C.c_void_p(stream))

    def work(self, ptr, n, stride=0):
        cnt = C.c_long()
        rc = self.L.qrl_pfb_work(self.h, C.c_void_p(ptr), n, stride, 1, C.byref(cnt))
        if rc:
            raise RuntimeError("qrl_pfb_work failed: %s" % self.L.qrl_last_error(self.h))
        return cnt.value

    def out(self):
        d, s, n = C.c_void_p(), C.c_long(), C.c_long()
        self.L.qrl_pfb_out_device(self.h, C.byref(d), C.byref(s), C.byref(n))
        return d.value, s.value, n.value

    def close(self):
        self.L.qrl_pfb_destroy(self.h)


class _DevRows:
    def __init__(self, ptr, rows, cols, stride):
        self.__cuda_array_interface__ = {"shape": (rows, cols), "strides": (8 * stride, 8), "typestr": "<c8", "data": (ptr, False),
                                         "version": 2}


def _kernel_ms(torch, fn, k):
    """device time per call of each pfb kernel, from a torch.profiler trace of k calls"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(k):
            fn()
        torch.cuda.synchronize()
    res = {}
    for e in prof.key_averages():
        for name in ("pfb_dft_kernel", "pfb_fir_kernel", "pfb_chan_kernel", "pfb_synth_kernel", "pfb_chan_generic_kernel",
                     "pfb_synth_generic_kernel", "pfb_tail_kernel", "pfb_synth_tail_kernel"):
            if name + "<" in e.key or name + "(" in e.key or e.key.endswith(name):
                us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                res[name] = res.get(name, 0.0) + us / 1e3 / k
    return res


def lowpass(L, gain, fs):
    buf = np.zeros(1 << 20, np.float32)
    n = L.qrl_firdes_low_pass_2(float(gain), float(fs), 5000.0, 2000.0, 60.0, 5, buf.ctypes.data_as(C.c_void_p), len(buf))
    assert n > 0
    return buf[:n].copy()


def shape_case(torch, dev, stream, libs, label, M, fs, ntaps, k, sm_count):
    L = libs[0][1]
    if ntaps is None:
        ctaps, staps = lowpass(L, 1, fs), lowpass(L, M, fs)
    else:
        ctaps = np.random.default_rng(100 + M).standard_normal(ntaps).astype(np.float32) / ntaps
        staps = ctaps * M
    tpf = (len(ctaps) + M - 1) // M
    cols = N_WIDE // M
    g = torch.Generator(device=dev).manual_seed(M)
    x = torch.view_as_complex(torch.randn((N_WIDE, 2), device=dev, generator=g) * 0.3)
    z = torch.view_as_complex(torch.randn((M, cols, 2), device=dev, generator=g) * 0.3)
    res = {"M": M, "fs_hz": fs, "taps": len(ctaps), "taps_per_branch": tpf, "wideband_samples_per_call": N_WIDE,
           "ffma_per_wideband_sample": 4 * M + 2 * tpf}
    for kind, name, taps, inp, n, stride in ((CHANNELIZER, "channelizer", ctaps, x, N_WIDE, 0), (SYNTHESIZER, "synthesizer", staps, z, cols, cols)):
        hs = [(tag, Pfb(Lx, kind, M, taps, n, stream.cuda_stream)) for tag, Lx in libs]
        outs = {}
        for tag, h in hs:                                                  # first call of each build: outputs compared bit for bit
            h.work(inp.data_ptr(), n, stride)
            p, s, items = h.out()
            o = torch.as_tensor(_DevRows(p, M, items, s), device=dev) if kind == CHANNELIZER else torch.as_tensor(_DevRows(p, 1, items, items), device=dev)
            outs[tag] = o.clone()
        runs = {tag: [] for tag, _ in hs}
        for _ in range(3):                                                 # alternated, so both builds see the same clocks and neighbours
            for tag, h in hs:
                runs[tag].append(timed_calls(lambda: h.work(inp.data_ptr(), n, stride), k, stream, torch, warm=2))
        sm_clk = _smi("clocks.sm")[0]
        r = {}
        for tag, h in hs:
            ms = float(np.median(runs[tag]))
            kms = _kernel_ms(torch, lambda: h.work(inp.data_ptr(), n, stride), k)
            e = {"ms_per_call": ms, "ms_per_call_runs": runs[tag], "gsamples_per_s": N_WIDE / (ms * 1e-3) / 1e9,
                 "x_realtime": N_WIDE / fs / (ms * 1e-3), "kernel_ms_per_call": kms}
            try:
                peak = sm_count * 128 * float(sm_clk) * 1e6
                e["call_ffma_issue_share"] = (4 * M + 2 * tpf) * N_WIDE / (ms * 1e-3) / peak
                if kms.get("pfb_dft_kernel"):
                    e["dft_kernel_ffma_issue_share"] = 4 * M * N_WIDE / (kms["pfb_dft_kernel"] * 1e-3) / peak
                if kms.get("pfb_fir_kernel"):
                    e["fir_kernel_ffma_issue_share"] = 2 * tpf * N_WIDE / (kms["pfb_fir_kernel"] * 1e-3) / peak
            except ValueError:
                pass
            r[tag] = e
        if len(hs) > 1:
            r["outputs_bit_identical_between_builds"] = bool(torch.equal(torch.view_as_real(outs[hs[0][0]]), torch.view_as_real(outs[hs[1][0]])))
            r["speedup_vs_" + hs[1][0]] = r[hs[1][0]]["ms_per_call"] / r[hs[0][0]]["ms_per_call"]
        r["sm_clock_sampled_mhz"] = sm_clk
        res[name] = r
        for _, h in hs:
            h.close()
        del outs
    del x, z
    torch.cuda.empty_cache()
    return res


def mmdvm_bank(torch, dev, stream, k):
    """10 Msps -> channelizer(400) -> qrl_mmdvm_rx over all 400 rows of its [400][stride] device output"""
    import qradiolink_b200 as q
    M, fs = 400, 10e6
    L = q.load_library()
    ch = q.PfbChannelizer(M, lowpass(L, 1, fs), max_in=N_WIDE)
    ch.set_stream(stream.cuda_stream)
    frames = N_WIDE // M + 1
    rx = q.MmdvmChannelsRx(M, rows=list(range(M)), n_rows=M, max_in=frames)
    rx.set_stream(stream.cuda_stream)
    g = torch.Generator(device=dev).manual_seed(400)
    x = torch.view_as_complex(torch.randn((N_WIDE, 2), device=dev, generator=g) * 0.3)

    def call():
        n = ch.work_device(x.data_ptr(), N_WIDE)
        p, s, _ = ch.out_device()
        rx.work_device(p, n, s)

    runs = [timed_calls(call, k, stream, torch, warm=2) for _ in range(3)]
    ms = float(np.median(runs))
    ch.close(); rx.close()
    return {"what": "10 Msps -> qrl_pfb channelizer M = 400 -> qrl_mmdvm_rx on all 400 rows (25 ksps -> int16 at 24 ksps)",
            "wideband_samples_per_call": N_WIDE, "ms_per_call": ms, "ms_per_call_runs": runs, "x_realtime": N_WIDE / fs / (ms * 1e-3),
            "sm_clock_sampled_mhz": _smi("clocks.sm")[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=5, help="timed calls per run")
    ap.add_argument("--lib", default=None, help="another libqrl_b200.so, timed on the same shapes alternately with this build")
    ap.add_argument("--only", default=None, help="comma-separated M values to run (default: all shapes)")
    args = ap.parse_args()
    import torch
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as QL
    q.load_library()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power, sm_max, sm_now = (_smi("name,power.limit,clocks.max.sm,clocks.sm") + ["?"] * 4)[:4]
    sm_count = torch.cuda.get_device_properties(dev).multi_processor_count
    libs = [("this_build", _open(QL._LIB_PATH))]
    if args.lib:
        libs.append(("other_build", _open(os.path.abspath(args.lib))))
    out = {"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": sm_max, "sm_clock_at_start_mhz": sm_now, "sm_count": sm_count,
           "other_build": os.path.abspath(args.lib) if args.lib else None}
    only = None if not args.only else {int(m) for m in args.only.split(",")}
    stream = torch.cuda.Stream(dev)
    with torch.cuda.stream(stream):
        for label, M, fs, ntaps in SHAPES:
            if only and M not in only:
                continue
            # shapes a build refuses (the parent takes M <= 64 only) are timed on this build alone
            use = libs if (M <= 64 or len(libs) == 1) else libs[:1]
            out[label] = shape_case(torch, dev, stream, use, label, M, fs, ntaps, args.k, sm_count)
        if not only or 400 in only:
            out["mmdvm_bank_400"] = mmdvm_bank(torch, dev, stream, args.k)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
