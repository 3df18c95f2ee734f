"""Throughput of the ccsds_ldpc_decoder path (rate 7/8 C2 code) on the GPU: the decoder alone on a device-resident soft stream.

Prints one JSON line: the card and its power limit (read in the same run), ms per push, codewords/s and info Gbit/s, the per-kernel event
times (correlation, frame walk, gather, decode + CADU repack) and the spread over the repeats. Every timed push's CADUs are checked against
the transmitted frames. The fused IQ -> CADU chain is not measured here (the synthetic transmitter has no LDPC signal configuration yet).

Usage: python tools/bench_ldpc.py [--log2-soft 28] [--repeats 5] [--iterations 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [v.strip() for v in out.splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e!r})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2-soft", type=int, default=28)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iterations", type=int, default=10)
    ap.add_argument("--unique", type=int, default=256, help="distinct codewords, tiled over the push")
    a = ap.parse_args()
    import torch
    from satdump_b200 import capi, synth
    tx, _, clear = synth.ldpc_frames(a.unique, 5)
    nfr = (1 << a.log2_soft) // 8192
    soft = synth.ldpc_soft(np.tile(tx, (nfr // a.unique + 1, 1))[:nfr].reshape(-1), "qpsk", sigma=12.0, seed=1)
    want = np.tile(clear, (nfr // a.unique + 1, 1))[:nfr]
    dev = torch.from_numpy(soft).cuda()
    f = capi.Fec(capi.ldpc_cfg("qpsk", ldpc_iterations=a.iterations, max_soft=soft.size))
    L = capi.lib()
    runs = []
    for r in range(a.repeats + 1):
        f._n = soft.size
        capi._chk(L.b200_fec_push_soft_device(f.h, dev.data_ptr(), soft.size))
        got = f.frames()
        # the last frame waits for the bytes of the next window unless its ASM is at its start
        bad = np.nonzero((got != want[:got.shape[0]]).any(1))[0]
        assert got.shape[0] >= nfr - 1 and bad.size == 0, f"{got.shape[0]} CADUs, {bad.size} differ from the transmitted frames: {bad[:8]}"
        if r:
            runs.append(dict(frames=int(got.shape[0]), **f.timing()))
        f = capi.Fec(capi.ldpc_cfg("qpsk", ldpc_iterations=a.iterations, max_soft=soft.size))  # a new stream per repeat
    push = np.array([x["push"] for x in runs])
    cw = np.array([x["frames"] for x in runs]) / (push / 1e3)
    name, power = card()
    print(json.dumps(dict(
        card=name, power_limit=power, soft_bytes_per_push=soft.size, iterations=a.iterations, repeats=a.repeats,
        ms_per_push=dict(median=float(np.median(push)), min=float(push.min()), max=float(push.max())),
        codewords_per_s=float(np.median(cw)), info_gbit_per_s=float(np.median(cw) * 7136 / 1e9),
        kernel_ms={k: float(np.median([x[k] for x in runs])) for k in ("corr", "walk", "gather", "decode")})))


if __name__ == "__main__":
    main()
