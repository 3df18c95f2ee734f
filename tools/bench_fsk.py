"""fsk_demod throughput on one GPU: BlueWalker3.json's bluewalker3_wide shape (512 ksym/s, rrc_alpha 0.35) at 2 MS/s cs16, 3.9 samples per
symbol, at 2^27 and 2^29 samples per push.

- device-resident: one push of samples already in HBM through the demodulator, fsk_demod and psk_demod BPSK (pll_bw 0.003) on the same
  samples, alternated, three rounds; per-stage device times from b200_demod_last_timing (front end + AGC + FIR, Costas, M&M);
- host to CADU: the fused chain (fsk_demod -> ccsds_conv_concat_decoder, bpsk_90, 9784-bit CADUs, no RS) fed from host memory.

The stream is a 2^24-sample synthetic signal repeated, so it has a discontinuity every 2^24 samples; the rates are what is measured.
Prints one JSON line with the card name and power limit beside the numbers.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    import torch
    from satdump_b200 import capi, synth
    fs, rs = 2_000_000, 512_000
    base, _ = synth.fsk_signal(1 << 24, fs, rs, h=0.7, seed=1, snr_db=12, fmt="cs16")
    out = {"card": card(), "shape": "bluewalker3_wide, 2 MS/s cs16", "sizes": {}}
    for logn in (27, 29):
        n = 1 << logn
        raw = np.tile(base, n >> 24)
        dev = torch.from_numpy(raw).cuda()
        res = {}
        demods = {"fsk_demod": capi.Demod(capi.fsk_demod_cfg(fs, rs, 0.35, fmt="cs16", max_batch=n)),
                  "psk_demod_bpsk": capi.Demod(capi.demod_cfg(fs, rs, "bpsk", 0.35, 0.003, "cs16", max_batch=n))}
        for k, d in demods.items():  # warm-up
            d.push_device(dev.data_ptr(), n)
        for _ in range(3):
            for k, d in demods.items():
                torch.cuda.synchronize()
                t = time.perf_counter()
                d.push_device(dev.data_ptr(), n)
                el = time.perf_counter() - t
                r = res.setdefault(k, {"MSps": [], "stage_ms": []})
                r["MSps"].append(round(n / el / 1e6, 1))
                r["stage_ms"].append({a: round(b, 2) for a, b in d.timing().items()})
        for d in demods.values():
            d.close()
        del demods
        ch = capi.Chain(capi.fsk_demod_cfg(fs, rs, 0.35, fmt="cs16", max_batch=n), capi.ccsds_cfg("bpsk_90", 9784, 0.3, 20, 0, max_soft=n))
        ch.push(raw)
        ch.frames()
        ch.reset()
        t = time.perf_counter()
        ch.push(raw)
        nf = ch.frames().size // (9784 // 8)
        el = time.perf_counter() - t
        res["fsk_chain_host_to_cadu"] = {"MSps": round(n / el / 1e6, 1), "cadus": int(nf)}
        ch.close()
        del dev
        out["sizes"][f"2^{logn}"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
