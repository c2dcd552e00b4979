"""Generates tests/golden/golden_freedv.json -- known-answer vectors of the FreeDV chains up to the codec2 modem boundary: outputs of
the CPU oracle (tests/freedv_oracle.c, qo_freedv_rx_* / qo_freedv_tx_*) on the seeded inputs of tests/golden/freedv_cases.py, recorded as
SHA-256 of their bytes + a few leading values (tests/golden/make_golden.py's format).

Run from the repo root:  python tests/golden/make_golden_freedv.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import freedv_oracle as O  # noqa: E402
from tests.golden import freedv_cases as F  # noqa: E402
from tests.golden.make_golden import describe, sha  # noqa: E402


def main():
    out = {"version": 1, "generator": "tests/golden/make_golden_freedv.py", "rx": {}, "tx": {}}
    for name, (sps, fs, _cf, fw, lo, sb) in F.RX_CASES.items():
        X = F.rx_signal(name)
        rec = {"input_sha256": sha(X), "channels": []}
        for c in range(X.shape[0]):
            p0, p1 = O.FreedvRx(sps, fs, fw, lo, sb).work(X[c])
            rec["channels"].append([describe(p0), describe(p1)])
        out["rx"][name] = rec
    for name, (sps, fs, _cf, fw, lo, sb) in F.TX_CASES.items():
        s = F.tx_input()
        out["tx"][name] = {"input_sha256": sha(s), "out": describe(O.FreedvTx(sps, fs, fw, lo, sb).work(s))}
    path = os.path.join(ROOT, "tests", "golden", "golden_freedv.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
