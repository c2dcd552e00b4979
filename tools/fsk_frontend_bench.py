"""The headline workload (64 channels of 4FSK-2k-FM, make_gr_demod_4fsk(5, 1e6, 1700, 3000, true), overlapped 2^22-sample calls on
bench.py's inputs) with the fused receive front end (fsk_fm_frontend_kernel, one launch per slice) against a twin created with
QRL_FSK_FRONTEND=0 (stage 1, channel filter and demodulator as three launches), alternated in one process.  Per pair of steps it
prints one JSON line per handle: ms per call, the stage-1 slot (the fused kernel, or the stage-1 FIR alone) and the symbol-sync stage
per call from qrl_rx_profile, and the median SM clock sampled in the step; once per run the card and its power limit.

    python tools/fsk_frontend_bench.py [--pairs 5] [--calls 64]
    python tools/fsk_frontend_bench.py --trace OUT_DIR     # one torch.profiler trace of each handle (a few calls) under OUT_DIR

Reuses bench.py's inputs and clock sampler; writes nothing except the traces."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CHANNELS, N_BASES, T_CALL, ClockSampler  # noqa: E402


def _smi(fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader,nounits"], capture_output=True,
                         text=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def make(q, fused, stream):
    if fused:
        os.environ.pop("QRL_FSK_FRONTEND", None)
    else:
        os.environ["QRL_FSK_FRONTEND"] = "0"
    try:
        blk = q.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=CHANNELS, max_samples=T_CALL)
    finally:
        os.environ.pop("QRL_FSK_FRONTEND", None)
    blk.set_stream(stream.cuda_stream)
    blk.set_overlap(True)
    return blk


def stage_ms(L, blk, stage):
    ms, n = C.c_double(), C.c_long()
    L.qrl_rx_profile_read(blk._h, stage, C.byref(ms), C.byref(n))
    return ms.value, n.value


def step(torch, L, blk, X, calls, stream, profile):
    """ms per call of `calls` back-to-back calls (tails joined inside the timed region), with the stage times when profiling"""
    torch.cuda.synchronize()
    L.qrl_rx_profile(blk._h, 1 if profile else 0)
    sampler = ClockSampler(0)
    sampler.start()
    sampler.ready.wait(10.0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sampler.armed = True
    e0.record(stream)
    for _ in range(calls):
        blk.work_device(X.data_ptr(), T_CALL, T_CALL)
    blk.join()
    e1.record(stream)
    torch.cuda.synchronize()
    sampler.armed = False
    sampler.stop_flag = True
    sampler.join()
    res = {"ms_per_call": e0.elapsed_time(e1) / calls,
           "sm_mhz_median": float(np.median(sampler.samples)) if sampler.samples else None}
    if profile:
        s0, n0 = stage_ms(L, blk, 0)
        s3, _ = stage_ms(L, blk, 3)
        res.update({"stage1_slot_ms_per_call": s0 / calls, "stage1_slot_launches_per_call": n0 / calls,
                    "symbol_sync_ms_per_call": s3 / calls})
    L.qrl_rx_profile(blk._h, 0)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=5)
    ap.add_argument("--calls", type=int, default=64)
    ap.add_argument("--trace", default=None, help="write one torch.profiler trace per handle under this directory instead")
    args = ap.parse_args()
    import torch
    import qradiolink_b200 as q
    from qradiolink_b200 import synth
    if q.device_count() < 1:
        raise SystemExit("fsk_frontend_bench.py: no CUDA device")
    dev = torch.device("cuda", 0)
    name, plimit, maxclk = _smi("name,power.limit,clocks.max.sm")
    print(json.dumps({"card": name, "power_limit_w": plimit, "sm_max_mhz": maxclk}), flush=True)
    bases = [synth.burst_4fsk(1000 + i, T_CALL) for i in range(N_BASES)]
    X = synth.batch_on_device(bases, CHANNELS, seed=4242, device=dev)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    L = q.load_library()
    handles = {"fused": make(q, True, stream), "three_launches": make(q, False, stream)}
    try:
        for blk in handles.values():
            for _ in range(4):
                blk.work_device(X.data_ptr(), T_CALL, T_CALL)
            blk.join()
        torch.cuda.synchronize()
        if args.trace:
            from torch.profiler import ProfilerActivity, profile
            os.makedirs(args.trace, exist_ok=True)
            for label, blk in handles.items():
                with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    for _ in range(6):
                        blk.work_device(X.data_ptr(), T_CALL, T_CALL)
                    blk.join()
                    torch.cuda.synchronize()
                path = os.path.join(args.trace, "fsk_frontend_%s.json" % label)
                prof.export_chrome_trace(path)
                print(json.dumps({"trace": path, "handle": label}), flush=True)
            return
        for p in range(args.pairs):
            for label, blk in handles.items():
                r = step(torch, L, blk, X, args.calls, stream, profile=False)
                r.update({k: v for k, v in step(torch, L, blk, X, 8, stream, profile=True).items() if k != "ms_per_call"
                          and k != "sm_mhz_median"})
                print(json.dumps(dict(pair=p, handle=label, **r)), flush=True)
    finally:
        for blk in handles.values():
            blk.close()


if __name__ == "__main__":
    main()
