"""Throughput of the metop_dump_decoder path (the MetOp X-band dump: QPSK, 35 Msym/s at 45 MS/s) on the GPU.

  decoder   the decoder alone on a device-resident soft stream: a locked stream (every window's ASM at position 0, so the frame walk
            takes up to 128 frames per round) and noise (every window shifts: one frame per round, the serial case)
  chain     the fused chain from cs16 IQ at the pipeline's parameters (synth.CONFIGS["metop_dump"]), device-resident input, synchronous
            pushes; GS/s and the real-time factor against 45 MS/s
  reference the reference's module loop (oracle/_ref/libsatref_dump.so) on one CPU thread of this host, on the same two soft streams;
            null where it was not built

Each timing is a host clock around calls that end in a device synchronise, after one warm-up call of the same shape. Prints one JSON line
with the card, its power limit and SM clock read in the same run. Every timed decoder push's CADUs are checked against the transmitted
frames. Of the chain's frames after the lock, the number whose message bytes are a transmitted frame's is reported (an RS failure at the
synthesised SNR leaves a frame's errors in place), and every repeat must write the same frames.

Usage: python tools/bench_metop_dump.py [--frames 4096] [--noise-frames 512] [--chain-log2 24] [--repeats 5] [--ref-frames 256]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

F = 8192
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
    return dict(s_median=float(np.median(t)), s_min=float(t.min()), s_max=float(t.max()), per_s=float(work / np.median(t)))


def time_decoder(soft, repeats, check=None):
    """seconds per push of the whole stream (one fresh decoder per push, device-resident input) and the frames of the last push"""
    import torch
    from satdump_b200 import capi
    dev = torch.from_numpy(soft).cuda()
    L = capi.lib()
    times, nf = [], 0
    for k in range(repeats + 1):
        f = capi.Fec(capi.dump_cfg(max_soft=soft.size))
        f._n = soft.size
        torch.cuda.synchronize()
        t = time.perf_counter()
        capi._chk(L.b200_fec_push_soft_device(f.h, dev.data_ptr(), soft.size))  # (returns after the decoder's stream synchronised)
        dt = time.perf_counter() - t
        got = f.frames()
        if check is not None:
            check(got)
        nf = got.shape[0]
        if k:
            times.append(dt)
        f.close()
    return times, nf


def reference_rate(soft, nframes):
    from oracle import dump as O
    if not O.available() or nframes <= 0:
        return None
    t = time.perf_counter()
    r = O.Dump().run(soft[:nframes * F + F // 2])
    return r["recs"].shape[0] / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096, help="frames of the locked stream per push")
    ap.add_argument("--noise-frames", type=int, default=512, help="frames of the noise stream per push")
    ap.add_argument("--chain-log2", type=int, default=24, help="log2 of the IQ samples per chain push")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--ref-frames", type=int, default=256, help="frames the reference decodes for its rate (0: skip it)")
    a = ap.parse_args()
    import torch
    from satdump_b200 import capi, synth
    out = dict(repeats=a.repeats)

    unique = 256
    tx, clear = synth.dump_frames(unique, seed=7)
    reps = a.frames // unique + 1
    locked = synth.dump_soft(np.tile(tx, (reps, 1))[:a.frames], 1, False, sigma=12.0, seed=1)
    want = np.tile(clear, (reps, 1))[:a.frames]

    def check_locked(got):
        assert got.shape[0] == a.frames and np.array_equal(got[:, :MSG], want[:, :MSG]), "locked stream: CADUs differ from the transmitted ones"

    t, nf = time_decoder(locked, a.repeats, check_locked)
    out["decoder_locked"] = dict(frames=nf, soft_bytes=int(locked.size), **stats(t, nf))
    noise = np.clip(np.round(np.random.default_rng(3).normal(0, 40, a.noise_frames * F)), -127, 127).astype(np.int8)
    t, nf = time_decoder(noise, a.repeats)
    out["decoder_noise"] = dict(frames=nf, soft_bytes=int(noise.size), **stats(t, nf))
    for k in ("decoder_locked", "decoder_noise"):
        out[k]["frames_per_s"] = out[k].pop("per_s")
        out[k]["soft_bytes_per_s"] = out[k]["soft_bytes"] / out[k]["s_median"]
    print(json.dumps(dict(progress={k: out[k] for k in ("decoder_locked", "decoder_noise")})), file=sys.stderr, flush=True)

    cfg = synth.CONFIGS["metop_dump"]
    n = 1 << a.chain_log2
    raw, clear_iq = synth.make_signal(cfg, n, seed=11, device="cuda")
    raw = raw.contiguous()
    ch = capi.Chain(capi.demod_cfg_for(cfg, max_batch=n), capi.fec_cfg_for(cfg, max_soft=2 * n + (1 << 20)))
    times, frames = [], []
    for k in range(a.repeats + 1):
        ch.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ch.push_device(raw.data_ptr(), n)
        got = ch.frames()
        dt = time.perf_counter() - t0
        if k:
            times.append(dt)
        frames.append(got)
    from tests.metop_dump_cases import after_lock
    tail = after_lock(frames[-1], clear_iq)
    sent = {row.tobytes() for row in clear_iq[:, :MSG]}
    ok = sum(row.tobytes() in sent for row in tail[:, :MSG])
    assert all(np.array_equal(f, frames[-1]) for f in frames) and ok >= 0.99 * tail.shape[0] > 0, f"chain: {ok} of {tail.shape[0]} frames"
    c = stats(times, n)
    out["chain_cs16"] = dict(samples=n, frames=int(frames[-1].shape[0]), frames_after_lock=int(tail.shape[0]), transmitted_message_bytes=ok,
                             s_median=c["s_median"], s_min=c["s_min"], s_max=c["s_max"], gsps=c["per_s"] / 1e9,
                             realtime_factor=c["per_s"] / cfg.samplerate)
    print(json.dumps(dict(progress=out["chain_cs16"])), file=sys.stderr, flush=True)

    out["reference_single_thread"] = dict(
        locked_frames_per_s=reference_rate(locked, a.ref_frames), noise_frames_per_s=reference_rate(noise, max(a.ref_frames // 8, 1) if a.ref_frames else 0),
        realtime_frames_per_s=cfg.symbolrate * 2 / F)
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
