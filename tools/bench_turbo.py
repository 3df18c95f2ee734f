"""Throughput of the ccsds_turbo_decoder path on the GPU: the decoder alone on a device-resident soft stream, for each (rate, base,
turbo_iters) combination the shipped pipelines use.

Prints one JSON line: the card, its power limit and SM clock (read in the same run), and per combination the ms per push, frames/s and
information Mbit/s on the device, the per-kernel event times (correlation, frame walk, gather, BCJR iterations, pack + CRC + compaction),
and the reference's single-thread frames/s on this host (oracle/_ref/libsatref_turbo.so, the module loop over a few frames; null where
it was not built). Every timed push's CADUs are checked against the transmitted frames.

Usage: python tools/bench_turbo.py [--frames 1024] [--repeats 3] [--ref-frames 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (turbo_rate, turbo_base, turbo_iters) of the shipped pipelines: Juice / Hera / Escapade ..., TGO, ORX, STEREO, Psyche, Chandrayaan-3
SHIPPED = [("1/2", 1115, 1), ("1/2", 1115, 5), ("1/2", 1115, 50), ("1/2", 223, 10), ("1/4", 1115, 2), ("1/6", 1115, 1), ("1/6", 1115, 20)]
RATE = {"1/2": 2, "1/4": 4, "1/6": 6}


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], text=True)
        name, power, sm, sm_max = [v.strip() for v in out.splitlines()[0].split(",")]
        return dict(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
    except Exception as e:  # noqa: BLE001
        return dict(card=f"unknown ({e!r})")


def reference_fps(rate, base, iters, soft, F, nframes):
    from oracle import turbo as O
    if not O.available():
        return None
    t = time.perf_counter()
    r = O.Turbo(rate, base, iters).run(soft[:nframes * F + 1])
    dt = time.perf_counter() - t
    return r["recs"].shape[0] / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024, help="frames per push (1024 = one decoding batch)")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--ref-frames", type=int, default=2, help="frames the reference decodes for its rate (0: skip it)")
    a = ap.parse_args()
    import torch
    from satdump_b200 import capi, synth
    out = dict(frames_per_push=a.frames, repeats=a.repeats, combos=[])
    for rate, base, iters in SHIPPED:
        r = RATE[rate]
        unique = 64
        tx, clear = synth.turbo_frames(unique, r, base, seed=7)
        F = tx.shape[1]
        reps = a.frames // unique + 1
        soft = synth.ldpc_soft(np.tile(tx, (reps, 1))[:a.frames].reshape(-1), "bpsk", sigma=30.0, seed=1)
        want = np.tile(clear, (reps, 1))[:a.frames]
        dev = torch.from_numpy(soft).cuda()
        L = capi.lib()
        runs = []
        for k in range(a.repeats + 1):  # the first push warms up
            f = capi.Fec(capi.turbo_cfg(rate, base, iters, max_soft=soft.size))
            f._n = soft.size
            capi._chk(L.b200_fec_push_soft_device(f.h, dev.data_ptr(), soft.size))
            got = f.frames()
            bad = np.nonzero((got != want[:got.shape[0]]).any(1))[0]
            assert got.shape[0] >= a.frames - 1 and bad.size == 0, f"{rate} {base} {iters}: {got.shape[0]} CADUs, {bad.size} differ"
            if k:
                runs.append(dict(frames=int(got.shape[0]), **f.turbo_timing()))
            f.close()
        push = np.array([x["push"] for x in runs])
        fps = np.array([x["frames"] for x in runs]) / (push / 1e3)
        ref = reference_fps(rate, base, iters, soft, F, a.ref_frames) if a.ref_frames else None
        out["combos"].append(dict(
            turbo_rate=rate, turbo_base=base, turbo_iters=iters, frame_soft_bytes=F,
            ms_per_push=dict(median=float(np.median(push)), min=float(push.min()), max=float(push.max())),
            frames_per_s=float(np.median(fps)), info_mbit_per_s=float(np.median(fps) * 8 * base / 1e6),
            kernel_ms={k: float(np.median([x[k] for x in runs])) for k in ("corr", "walk", "gather", "bcjr", "pack")},
            reference_single_thread_frames_per_s=ref))
        print(json.dumps(dict(progress=out["combos"][-1])), file=sys.stderr, flush=True)
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
