"""M17 frame codec throughput on one GPU: qrl_m17_rx_work (decode) and qrl_m17_tx_work (encode) at 4096 channels x 64 frames per call,
inputs resident in HBM, timed with CUDA events.  Prints one JSON line with frames per second, the card's name and power limit, and
the compiled reference codec's single-core frames per second (oracle/_ref/libqrl_ref_m17.so, where it was built).

    python tools/m17_codec_bench.py [--channels 4096] [--frames 64] [--iters 20]

Writes nothing."""
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

from qradiolink_b200 import m17 as Q  # noqa: E402
from tests import m17_model as M  # noqa: E402
from tests import test_m17_codec as T  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return "unknown", "unknown"


def records(Cn, F):
    """a transmission's LSF frame and stream frames, tiled over the channels: [Cn][F][56] deframer records"""
    tx = M.Transmitter()
    tx.set_lsf(Q.m17_lsf("N0CALL", "W1AW", 1, 0))
    rng = np.random.default_rng(7)
    frames = [(M.LSF, tx.step(1, None)[50:])] + [(M.STREAM, tx.step(2, rng.bytes(16))[2:48]) for _ in range(F - 1)]
    one = np.zeros((F, 56), np.uint8)
    for f, (t, p) in enumerate(frames):
        one[f, :4] = np.frombuffer(np.uint32(t).tobytes(), np.uint8)
        one[f, 4:8] = np.frombuffer(np.uint32(46).tobytes(), np.uint8)
        one[f, 8:54] = np.frombuffer(p, np.uint8)
    return np.ascontiguousarray(np.broadcast_to(one, (Cn, F, 56))), frames


def timed(torch, stream, fn, iters):
    """device time per call: events on the stream the handle runs on, around `iters` calls after one warm-up call"""
    assert fn() == 0
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(iters):
        assert fn() == 0
    b.record(stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=4096)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    L = Q.load_library()
    Cn, F = a.channels, a.frames
    stream = torch.cuda.Stream()
    rec_h, frames = records(Cn, F)
    rec = torch.from_numpy(rec_h).cuda()
    cnt = torch.full((Cn,), F, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    dec = Q.M17Decoder(Cn, F)
    dec.set_stream(stream.cuda_stream)
    rx_ms = timed(torch, stream, lambda: L.qrl_m17_rx_work(dec._h, C.c_void_p(rec.data_ptr()), C.c_void_p(cnt.data_ptr()), 56, F, 1), a.iters)
    check = Q.M17Decoder(Cn, F)                      # the timed calls carried state from call to call: check one fresh call
    check.set_stream(stream.cuda_stream)
    assert L.qrl_m17_rx_work(check._h, C.c_void_p(rec.data_ptr()), C.c_void_p(cnt.data_ptr()), 56, F, 1) == 0
    got = check.read()
    want = M.Decoder().work(frames)
    assert T.snapshots(got[0]) == want and T.snapshots(got[-1]) == want, "decoder output differs from the restatement"

    enc = Q.M17Encoder(Cn, F)
    enc.set_stream(stream.cuda_stream)
    for c in range(Cn):
        enc.set_lsf(c, Q.m17_lsf("N0CALL"))
    ops = torch.full((Cn, F), Q.OP_STREAM, dtype=torch.uint8, device="cuda")
    pl = torch.randint(0, 256, (Cn, F, 16), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    tx_ms = timed(torch, stream, lambda: L.qrl_m17_tx_work(enc._h, C.c_void_p(ops.data_ptr()), C.c_void_p(pl.data_ptr()), F, 1), a.iters)

    res = {"metric": "m17_codec", "channels": Cn, "frames_per_call": F, "decode_ms_per_call": round(rx_ms, 4),
           "decode_frames_per_s": round(Cn * F / rx_ms * 1e3), "encode_ms_per_call": round(tx_ms, 4),
           "encode_frames_per_s": round(Cn * F / tx_ms * 1e3)}
    res["gpu"], res["power_limit"] = card()
    R = T.ref_m17()
    if R is None:
        res["ref_single_core_decode_frames_per_s"] = res["ref_single_core_encode_frames_per_s"] = "not measured (oracle/_ref absent)"
    else:
        recs = frames * 50
        t0 = time.perf_counter(); T.ref_decode(R, recs); t1 = time.perf_counter()
        res["ref_single_core_decode_frames_per_s"] = round(len(recs) / (t1 - t0))
        n = 3000
        ops_h = np.array([1] + [2] * (n - 1), np.uint8); pl_h = np.zeros((n, 16), np.uint8)
        t0 = time.perf_counter(); T.ref_transmit(R, ("N0CALL", "", 0, 0), ops_h, pl_h); t1 = time.perf_counter()
        res["ref_single_core_encode_frames_per_s"] = round(n / (t1 - t0))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
