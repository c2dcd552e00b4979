"""DMR burst decoder throughput: 4096 channels x 2^16 bits per call, in HBM, both slots carrying voice superframes (AMBE FEC on) and
data bursts with bit errors.  Prints one JSON line: decode ms per call and bursts/s from CUDA events after warm-up, the card's name and
power limit read in the same run, and the compiled reference's bursts/s on one host core (oracle/_ref/libqrl_ref_dmr.so, when built)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=4096)
    ap.add_argument("--bits", type=int, default=1 << 16)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    import qradiolink_b200 as q
    from tests import dmr_model as M
    rng = np.random.default_rng(1)
    pool = []
    while sum(len(p) for p in pool) < 8 * a.bits:
        pool.append(M.mixed_stream(rng, 40, errors=(0, 1, 2, 3)))
    pool = np.concatenate(pool)
    rows = np.stack([np.roll(pool, 4099 * c)[:a.bits] for c in range(64)])
    bits = torch.from_numpy(rows[np.arange(a.channels) % 64]).cuda()
    counts = torch.full((a.channels,), a.bits, dtype=torch.int32, device="cuda")
    dec = q.DmrBurstDecoder(a.channels, a.bits, a.bits // 288 + 2, ambe_fec=True)
    L = q.load_library()
    s = torch.cuda.Stream()         # a stream of its own: set_stream(NULL) would mean "back to the handle's own stream"
    dec.set_stream(s.cuda_stream)

    def call():
        q.lib.check(L.qrl_dmr_rx_work(dec._h, C.c_void_p(bits.data_ptr()), C.c_void_p(counts.data_ptr()), a.bits, 1), dec._h, "work")

    for _ in range(3):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(a.iters):
        call()
    e1.record(s)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.iters
    n_bursts = int(sum(len(r) for r in dec.read()))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    ref_rate = None
    lib = os.path.join(ROOT, "oracle", "_ref", "libqrl_ref_dmr.so")
    if os.path.exists(lib):
        R = C.CDLL(lib)
        R.ref_dmr_create.restype = C.c_void_p
        h = C.c_void_p(R.ref_dmr_create())
        row = np.ascontiguousarray(rows[0], np.uint8)
        out = np.zeros((a.bits // 288 + 2, 72), np.uint8)
        ch = np.array([a.bits], np.int32)
        t = time.perf_counter()
        n = R.ref_dmr_work(h, row.ctypes.data_as(C.c_void_p), C.c_long(len(row)), ch.ctypes.data_as(C.c_void_p), 1, 1,
                           out.ctypes.data_as(C.c_void_p), len(out))
        ref_rate = n / (time.perf_counter() - t)
        R.ref_dmr_destroy(h)
    print(json.dumps({"channels": a.channels, "bits_per_call": a.bits, "decode_ms_per_call": round(ms, 4),
                      "bursts_per_call": n_bursts, "bursts_per_s": round(n_bursts / (ms / 1e3)), "gpu": gpu,
                      "ref_bursts_per_s_one_core": None if ref_rate is None else round(ref_rate)}))


if __name__ == "__main__":
    main()
