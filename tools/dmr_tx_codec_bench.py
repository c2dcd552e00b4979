"""DMR burst encoder throughput: 4096 channels x 64 ops per call, ops and vocoder frames in HBM, in steady voice after a header; every
16th channel starts each call with a header and ends it with a stop and the audio that brings the terminator.  Prints one JSON line:
encode ms per call, bursts/s and output GB/s (72 bytes per burst) from CUDA events after warm-up, the card's name, power limit and SM
clock read in the same run, and the compiled reference encoders' voice bursts/s on one host core (oracle/_ref/libqrl_ref_dmr_tx.so,
when built)."""
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
    ap.add_argument("--ops", type=int, default=64)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    import torch
    import qradiolink_b200 as q
    from qradiolink_b200 import dmr as D
    rng = np.random.default_rng(1)
    ops = np.full((a.channels, a.ops), D.OP_AUDIO, np.uint8)
    ops[::16, 0] = D.OP_HEADER
    ops[::16, a.ops - 7] = D.OP_STOP
    audio = rng.integers(0, 256, (a.channels, a.ops, 9)).astype(np.uint8)
    enc = q.DmrBurstEncoder(a.channels, a.ops)
    enc.set_config(color_code=3, timeslot=1, src_id=2342, dst_id=91, talker_alias="BENCH ALIAS 0123456789")
    enc.reset()
    head = ops.copy()
    head[:, 0] = D.OP_HEADER
    enc.work(head, audio, collect=False)                # every channel active
    d_ops, d_audio = torch.from_numpy(ops).cuda(), torch.from_numpy(audio).cuda()
    s = torch.cuda.Stream()         # a stream of its own: set_stream(NULL) would mean "back to the handle's own stream"
    enc.set_stream(s.cuda_stream)
    torch.cuda.synchronize()
    for _ in range(5):
        enc.work_device(d_ops.data_ptr(), d_audio.data_ptr(), a.ops)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(a.iters):
        enc.work_device(d_ops.data_ptr(), d_audio.data_ptr(), a.ops)
    e1.record(s)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.iters
    _, recs = enc.read()
    n_bursts = int(sum(len(r) for r in recs))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ref_rate = None
    lib = os.path.join(ROOT, "oracle", "_ref", "libqrl_ref_dmr_tx.so")
    if os.path.exists(lib):
        R = C.CDLL(lib)
        o = np.zeros(33, np.uint8)
        au = np.ascontiguousarray(audio[0, :3].reshape(-1))
        n = 20000
        t = time.perf_counter()
        for k in range(n):
            R.ref_dmr_tx_voice(au.ctypes.data_as(C.c_void_p), k % 6, 3, 0, 0xC2, 0, C.c_uint(2342), C.c_uint(91), o.ctypes.data_as(C.c_void_p))
        ref_rate = n / (time.perf_counter() - t)
    print(json.dumps({"channels": a.channels, "ops_per_call": a.ops, "encode_ms_per_call": round(ms, 4), "bursts_per_call": n_bursts,
                      "bursts_per_s": round(n_bursts / (ms / 1e3)), "out_GB_per_s": round(n_bursts * 72 / (ms / 1e3) / 1e9, 2),
                      "gpu": gpu, "ref_voice_bursts_per_s_one_core": None if ref_rate is None else round(ref_rate)}))
    enc.close()


if __name__ == "__main__":
    main()
