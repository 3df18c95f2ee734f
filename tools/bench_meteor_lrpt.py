"""Throughput of meteor_lrpt_decoder (m2x_mode false, the METEOR M2 LRPT 72k pipeline's decoder) on the GPU.

  decoder   the decoder alone on a device-resident soft stream: a locked stream (every window's ASM at position 0, so the frame walk
            takes up to 128 frames per round and the Viterbi kernels decode them all at once) and noise (every window shifts: one frame
            per walk round, the serial case)
  reference the reference's module loop (oracle/_ref/libsatref_meteor.so) on one CPU thread of this host, on the same two soft streams;
            null where it was not built

Each timing is a host clock around calls that end in a device synchronise, after one warm-up call of the same shape. Prints one JSON line
with the card, its power limit and SM clock read in the same run. Every timed push of the locked stream is checked against the transmitted
frames (the frames whose derandomised byte 9 is 0xFF come out inverted, as the reference writes them).

Usage: python tools/bench_meteor_lrpt.py [--frames 4096] [--noise-frames 256] [--repeats 5] [--ref-frames 128]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

F = 16384
MSG = 4 + 4 * 223


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], text=True)
        name, power, sm, sm_max = [v.strip() for v in out.splitlines()[0].split(",")]
        return dict(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
    except Exception as e:  # noqa: BLE001
        return dict(card=f"unknown ({e!r})")


def stats(times, work):
    t = np.array(times)
    return dict(s_median=float(np.median(t)), s_min=float(t.min()), s_max=float(t.max()), frames_per_s=float(work / np.median(t)))


def time_decoder(soft, repeats, check=None):
    """seconds per push of the whole stream (one fresh decoder per push, device-resident input) and the frames walked in the last push"""
    import torch
    from satdump_b200 import capi
    dev = torch.from_numpy(soft).cuda()
    L = capi.lib()
    times, nf = [], 0
    for k in range(repeats + 1):
        f = capi.Fec(capi.meteor_lrpt_cfg(False, max_soft=soft.size))
        f._n = soft.size
        torch.cuda.synchronize()
        t = time.perf_counter()
        capi._chk(L.b200_fec_push_soft_device(f.h, dev.data_ptr(), soft.size))  # (returns after the decoder's stream synchronised)
        dt = time.perf_counter() - t
        got = f.frames()
        if check is not None:
            check(got)
        nf = f.meteor_frames().shape[0]
        if k:
            times.append(dt)
        f.close()
    return times, nf


def reference_rate(soft, nframes):
    from oracle import meteor as O
    if not O.available() or nframes <= 0:
        return None
    t = time.perf_counter()
    r = O.Meteor(False).run(soft[:nframes * F + F // 2])
    return r["recs"].shape[0] / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096, help="frames of the locked stream per push")
    ap.add_argument("--noise-frames", type=int, default=256, help="frames of the noise stream per push")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--ref-frames", type=int, default=128, help="frames the reference decodes for its rate (0: skip it)")
    a = ap.parse_args()
    from satdump_b200 import synth
    out = dict(repeats=a.repeats)
    coded, written = synth.lrpt_frames(a.frames, seed=7)
    locked = synth.lrpt_soft(coded, 1, False, sigma=30.0, seed=1)
    inv = written[:, 9] == 0xFF

    def check_locked(got):
        assert got.shape[0] == a.frames, got.shape
        assert np.array_equal(got[~inv, :MSG], written[~inv, :MSG]) and np.array_equal(got[inv, 4:MSG], written[inv, 4:MSG] ^ 0xFF), \
            "locked stream: CADUs differ from the transmitted ones"

    t, nf = time_decoder(locked, a.repeats, check_locked)
    out["decoder_locked"] = dict(frames=nf, soft_bytes=int(locked.size), **stats(t, nf))
    noise = np.clip(np.round(np.random.default_rng(3).normal(0, 40, a.noise_frames * F)), -127, 127).astype(np.int8)
    t, nf = time_decoder(noise, a.repeats)
    out["decoder_noise"] = dict(frames=nf, soft_bytes=int(noise.size), **stats(t, nf))
    for k in ("decoder_locked", "decoder_noise"):
        out[k]["soft_bytes_per_s"] = out[k]["soft_bytes"] / out[k]["s_median"]
    out["reference_single_thread"] = dict(
        locked_frames_per_s=reference_rate(locked, a.ref_frames), noise_frames_per_s=reference_rate(noise, max(a.ref_frames // 8, 1) if a.ref_frames else 0),
        realtime_frames_per_s=72000 * 2 / F)
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
