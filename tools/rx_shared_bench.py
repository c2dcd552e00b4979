"""Receive chains fed one 1 Msps SDR stream (qrl_rx_work / _sc16 / _sc8 with stride 0: one source, C receivers at C carrier offsets)
against the same call on C identical rows.  Workloads: 64 channels at 2^22 samples per call, channels at distinct offsets across
+-450 kHz, for 4FSK-2k-FM (stage 1 /50), NBFM (/125), QPSK-250K (/2: rotator pass) and the other register-tiled stage-1 shapes
(4FSK-1k-FM /100, 2FSK-2k-FM /25, QPSK-20K /25 with 681 taps, QPSK-2K /100 with 2727 taps).  Prints one JSON line with, per workload:
  * ms per call from HBM: stride 0 on one [T] capture against a [64][T] slab of identical rows, alternating in the same process;
  * stage-1 device time per call (qrl_rx_profile stage 0) on both, from HBM;
  * a bit-for-bit check of every port of three channels between the two on the first call;
  * for 4FSK-2k-FM, NBFM and QPSK-250K: ms per call from pinned host memory, stride 0 against identical rows, for gr_complex, sc16
    and sc8 input;
with the card, its power limit and the SM clocks.

    python tools/rx_shared_bench.py [--T 4194304] [--rounds 5] [--k 5]

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

WORKLOADS = {
    "4fsk_2k_fm": lambda q, n, m, dev: q.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=n, max_samples=m, device=dev),
    "nbfm": lambda q, n, m, dev: q.make_gr_demod_nbfm(125, 1000000, 1700, 5000, n_channels=n, max_samples=m, device=dev),
    "qpsk_250k": lambda q, n, m, dev: q.make_gr_demod_qpsk(2, 1000000, 1700, 160000, n_channels=n, max_samples=m, device=dev),
    # the other register-tiled stage-1 shapes (no host-fed runs): /100 with 9 taps per branch, /25 with 9 and 28, /100 with 28
    "4fsk_1k_fm": lambda q, n, m, dev: q.make_gr_demod_4fsk(10, 1000000, 1700, 2000, True, n_channels=n, max_samples=m, device=dev),
    "2fsk_2k_fm": lambda q, n, m, dev: q.make_gr_demod_2fsk(5, 1000000, 1700, 4000, True, n_channels=n, max_samples=m, device=dev),
    "qpsk_20k": lambda q, n, m, dev: q.make_gr_demod_qpsk(25, 1000000, 1700, 6500, n_channels=n, max_samples=m, device=dev),
    "qpsk_2k": lambda q, n, m, dev: q.make_gr_demod_qpsk(125, 1000000, 1700, 1300, n_channels=n, max_samples=m, device=dev),
}
HOST_FED = ("4fsk_2k_fm", "nbfm", "qpsk_250k")


def _smi(fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader,nounits"], capture_output=True,
                         text=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def _stage1_ms(L, blk, fn, k, torch):
    """stage-1 device time per call (qrl_rx_profile stage 0) over k calls"""
    torch.cuda.synchronize()
    L.qrl_rx_profile(blk._h, 1)
    for _ in range(k):
        fn()
    ms, n = C.c_double(), C.c_long()
    L.qrl_rx_profile_read(blk._h, 0, C.byref(ms), C.byref(n))
    L.qrl_rx_profile(blk._h, 0)
    return ms.value / k


def _median_alternating(fns, rounds, k, stream, torch):
    """median ms per call of each function, the functions timed in turn within every round"""
    t = [[] for _ in fns]
    for _ in range(rounds):
        for i, fn in enumerate(fns):
            t[i].append(timed_calls(fn, k, stream, torch, warm=1))
    return [float(np.median(x)) for x in t], t


def workload(q, torch, dev, name, Cn, T, rounds, k):
    L = q.load_library()
    stream = torch.cuda.current_stream()
    torch.cuda.empty_cache()
    t = torch.arange(T, device=dev, dtype=torch.float64)
    X = torch.zeros(T, device=dev, dtype=torch.complex64)
    for f in (-0.41, -0.17, 0.05, 0.29, 0.44):
        X += (0.15 * torch.polar(torch.ones_like(t), 2 * np.pi * f * t)).to(torch.complex64)
    X += torch.view_as_complex(torch.randn((T, 2), device=dev) * 0.05)
    del t
    slab = X[None, :].expand(Cn, T).contiguous()
    offsets = [(-0.45 + 0.9 * c / Cn) * 1e6 for c in range(Cn)]
    blks = [WORKLOADS[name](q, Cn, T, dev.index) for _ in range(2)]
    for b in blks:
        b.set_stream(stream.cuda_stream)
        for c, hz in enumerate(offsets):
            b.set_carrier_offset(hz, channel=c)
    # paths: stride 0 on one [T] capture, and a [Cn][T] slab of identical rows
    paths = {"shared": lambda: blks[0].work_device(X.data_ptr(), T, 0),
             "rows": lambda: blks[1].work_device(slab.data_ptr(), T, T)}
    owner = {"shared": blks[0], "rows": blks[1]}
    # parity on the first call of each handle: every port of three channels, bit for bit
    for fn in paths.values():
        fn()
    chans = [0, Cn // 2, Cn - 1]
    same = True
    for p in range(blks[0].nports):
        ref = blks[1].read_port(p)
        got = blks[0].read_port(p)
        same = same and all(got[c].tobytes() == ref[c].tobytes() for c in chans)
    names = list(paths)
    ms, rounds_ms = _median_alternating([paths[n] for n in names], rounds, k, stream, torch)
    st1 = {n: _stage1_ms(L, owner[n], paths[n], k, torch) for n in names}
    res = {"channels": Cn, "samples_per_channel_per_call": T, "parity_3_channels_all_ports": bool(same),
           "hbm_ms_per_call": dict(zip(names, ms)), "hbm_rounds": dict(zip(names, rounds_ms)),
           "rows_over_shared": ms[1] / ms[0], "shared_realtime_factor_per_channel": T / (ms[0] * 1e-3) / 1e6,
           "stage1_ms_per_call": st1}
    sh, rw = blks
    if name not in HOST_FED:
        sh.close(); rw.close()
        return res
    del slab, X
    torch.cuda.empty_cache()
    # host-fed: one pinned stream of T samples against a pinned [Cn][T] slab of identical rows
    rng = np.random.default_rng(1)
    x = (0.3 * (rng.standard_normal(T) + 1j * rng.standard_normal(T))).astype(np.complex64)
    host = {}
    for fmt in ("gr_complex", "sc16", "sc8"):
        if fmt == "gr_complex":
            one = torch.from_numpy(x.view(np.float32)).pin_memory()
            fn, scale = L.qrl_rx_work, None
        else:
            sc, top, dt = (16000.0, 32767, np.int16) if fmt == "sc16" else (90.0, 127, np.int8)
            w = np.clip(np.rint(x.view(np.float32) * sc), -top, top).astype(dt)
            one = torch.from_numpy(w).pin_memory()
            fn, scale = (L.qrl_rx_work_sc16 if fmt == "sc16" else L.qrl_rx_work_sc8), C.c_float(1.0 / sc)
        many = one[None, :].expand(Cn, one.shape[0]).contiguous().pin_memory()
        args = (lambda p, s: (sh._h, C.c_void_p(p), T, s, 0)) if scale is None else (lambda p, s: (sh._h, C.c_void_p(p), T, s, scale, 0))
        argr = (lambda p, s: (rw._h, C.c_void_p(p), T, s, 0)) if scale is None else (lambda p, s: (rw._h, C.c_void_p(p), T, s, scale, 0))
        a_sh, a_rw = args(one.data_ptr(), 0), argr(many.data_ptr(), T)
        call_s = lambda: fn(*a_sh)                                    # noqa: E731
        call_r = lambda: fn(*a_rw)                                    # noqa: E731
        (hs, hr), _ = _median_alternating([call_s, call_r], rounds, k, stream, torch)
        bytes_s = one.numel() * one.element_size()
        host[fmt] = {"shared_ms_per_call": hs, "rows_ms_per_call": hr, "rows_over_shared": hr / hs,
                     "h2d_bytes_per_call": {"shared": bytes_s, "rows": bytes_s * Cn}}
        del one, many
    res["pinned_host"] = host
    sh.close(); rw.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=1 << 22, help="samples per call at 1 Msps")
    ap.add_argument("--channels", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of the shared and the identical-rows path")
    ap.add_argument("--k", type=int, default=5, help="calls per timed round")
    args = ap.parse_args()
    import torch
    import qradiolink_b200 as q
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power, sm_max, sm_now = (_smi("name,power.limit,clocks.max.sm,clocks.sm") + ["?"] * 4)[:4]
    out = {"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": sm_max, "sm_clock_at_start_mhz": sm_now}
    # the handles run on a real torch stream (a NULL stream handle would give each its own, which the timing events do not see)
    with torch.cuda.stream(torch.cuda.Stream(dev)):
        for wl in WORKLOADS:
            out[wl] = workload(q, torch, dev, wl, args.channels, args.T, args.rounds, args.k)
    out["sm_clock_at_end_mhz"] = _smi("clocks.sm")[0]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
