"""Throughput of the FengYun-3 decoders behind psk_demod QPSK on the GPU: fengyun_ahrpt_decoder (--decoder ahrpt, the AHRPT / DPT
pipelines) or fengyun_mpt_decoder (--decoder mpt, the A/B/C MPT pipeline).

  decoder    the decoder alone on a locked soft stream of --soft-log2 bytes already in device memory (b200_fec_push_soft_device), in Msym/s
             (one symbol = one soft pair), and the device time of each kernel of one such push (torch.profiler, in a separate run)
  chain      IQ -> psk_demod QPSK -> the decoder through the fused chain, synchronous, one push of --chain-log2 samples. ahrpt: the
             FY-3E / F / H shape (QPSK 38.4 Msym/s, cs16 at 76.8 MS/s, invert_second_viterbi); mpt: the MPT shape (QPSK 18.7 Msym/s,
             cs16 at 40 MS/s)
  reference  the reference's module loop (oracle/_ref/libsatref_fengyun.so or libsatref_fengyun_mpt.so, 16384-byte reads) on one CPU
             thread of this host, on the first 2^24 bytes of the same locked stream; null where it was not built

Each timing is a host clock around one push, which returns after its frames are written on the device (the pull to the host and the
check are outside it), after one warm-up push of the same shape; the median of --repeats. Prints one JSON line with the card, its power
limit and SM clock read in the same run. Every timed push's CADUs are checked against the transmitted frames. Real time is 76.8e6 soft
bytes/s at 38.4 Msym/s (ahrpt) and 37.4e6 at 18.7 Msym/s (mpt).

Usage: python tools/bench_fengyun.py [--decoder ahrpt|mpt] [--soft-log2 28] [--repeats 5] [--chain-log2 24]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SYMRATE = {"ahrpt": 38.4e6, "mpt": 18.7e6}  # FY-3E / F / H AHRPT, FY-3A / B / C MPT
RT_KEY = {"ahrpt": "x_realtime_38M4", "mpt": "x_realtime_18M7"}
CHAIN = {"ahrpt": ("fengyun_ahrpt_e", "chain_fy3e"), "mpt": ("fengyun_mpt", "chain_mpt")}  # signal config, result key


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], text=True)
        name, power, sm, sm_max = [v.strip() for v in out.splitlines()[0].split(",")]
        return dict(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
    except Exception as e:  # noqa: BLE001
        return dict(card=f"unknown ({e!r})")


def timed(push, pull, repeats):
    """median seconds of push() over `repeats` calls after a warm-up one; pull() follows every call, untimed"""
    push()
    pull()
    t = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        push()
        t.append(time.perf_counter() - t0)
        pull()
    return float(np.median(t))


def locked_stream(nbytes, decoder):
    """nbytes of soft pairs carrying CADUs from the stream's first read (ahrpt: with invert_second_viterbi), and the CADUs"""
    from satdump_b200 import synth
    if decoder == "mpt":  # 8192 CADU bits = 4096 pairs of branch bits, 8192 symbols per branch
        i_bits, q_bits, clear = synth.fengyun_mpt_frames(nbytes // 16384 + 2, seed=1)
        soft = lambda i, q, seed: synth.fengyun_mpt_soft(i, q, sigma=12.0, seed=seed)  # noqa: E731
    else:  # 8192 CADU bits = 4096 pairs of branch bits, 4096 * 4 / 3 symbols per branch
        i_bits, q_bits, clear = synth.fengyun_frames(int(nbytes / 2 / (8192 * 2 / 3)) + 2, seed=1)
        soft = lambda i, q, seed: synth.fengyun_soft(i, q, sigma=12.0, seed=seed, invert_second=True)  # noqa: E731
    out = np.empty(nbytes, np.int8)
    step = 1 << 24
    for a in range(0, nbytes, step):  # (in slices, to bound the float temporaries)
        b = min(nbytes, a + step)
        out[a:b] = soft(i_bits[a // 2:b // 2], q_bits[a // 2:b // 2], a)
    return out, clear


def check(got, sent_set, what):
    good = sum(bytes(x) in sent_set for x in got)
    assert got.shape[0] > 0 and good >= got.shape[0] - 2, f"{what}: {good} of {got.shape[0]} CADUs were sent"


def kernel_times(f, dev_soft, n, outdir):
    """device ms per kernel name over one push (torch.profiler with CUDA activities), and the trace under outdir"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f.push_device(dev_soft, n)
        torch.cuda.synchronize()
    f.frames()
    ms = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.key.startswith(("k_", "void b200", "void k_")) or "b200::" in e.key:
            name = e.key.split("(")[0].replace("void ", "").replace("b200::", "")
            ms[name] = ms.get(name, 0.0) + e.device_time_total / 1e3
    if outdir:
        prof.export_chrome_trace(os.path.join(outdir, "bench_fengyun.pt.trace.json"))
    return {k: round(v, 3) for k, v in sorted(ms.items(), key=lambda kv: -kv[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--decoder", choices=["ahrpt", "mpt"], default="ahrpt")
    ap.add_argument("--soft-log2", type=int, default=28)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--chain-log2", type=int, default=24)
    ap.add_argument("--trace-dir", default=None, help="where the profiler trace goes (default: a temporary directory, removed)")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    from satdump_b200 import capi, synth
    if a.decoder == "mpt":
        from oracle import fengyun_mpt as O
        cfg_for, ref_for = (lambda n: capi.fengyun_mpt_cfg(20, 0.3, max_soft=n)), (lambda: O.RefMpt(20, 0.3))
    else:
        from oracle import fengyun as O
        cfg_for, ref_for = (lambda n: capi.fengyun_ahrpt_cfg(20, 0.26, True, max_soft=n)), (lambda: O.Ref(20, 0.26, True))
    symrate, rt_key = SYMRATE[a.decoder], RT_KEY[a.decoder]
    res = dict(card(), decoder_kind=a.decoder)
    n = 1 << a.soft_log2
    soft, sent = locked_stream(n, a.decoder)
    dev = torch.from_numpy(soft).cuda()
    f = capi.Fec(cfg_for(n))
    sent = {bytes(x) for x in sent}
    # (each push continues the stream; the first one locks, the later ones stay locked)
    t = timed(lambda: f.push_device(dev.data_ptr(), n), lambda: check(f.frames(), sent, "decoder push"), a.repeats)
    res["decoder"] = dict(soft_bytes=n, Msym_per_s=n / 2 / t / 1e6, **{rt_key: n / 2 / t / symrate}, ms_per_push=t * 1e3)
    with tempfile.TemporaryDirectory() as tmp:
        res["decoder"]["kernel_ms_per_push"] = kernel_times(f, dev.data_ptr(), n, a.trace_dir or tmp)
    f.close()
    del dev
    sig = synth.CONFIGS[CHAIN[a.decoder][0]]
    ns = 1 << a.chain_log2
    raw, clear = synth.make_signal(sig, ns, seed=5, device="cuda")
    raw = raw.cpu().numpy()
    ch = capi.Chain(capi.demod_cfg_for(sig, max_batch=ns), capi.fec_cfg_for(sig, max_soft=ns))
    clear = {bytes(x) for x in clear}

    def pull():
        check(ch.frames(), clear, "chain push")
        ch.reset()

    t_chain = timed(lambda: ch.push(raw), pull, a.repeats)
    ch.close()
    res[CHAIN[a.decoder][1]] = dict(samples=ns, MSps=ns / t_chain / 1e6, Msym_per_s=ns / t_chain / (sig.samplerate / sig.symbolrate) / 1e6,
                                    x_realtime=ns / t_chain / sig.samplerate)
    if O.available():
        m = min(n, 1 << 24)
        ref = ref_for()
        t0 = time.perf_counter()
        r = ref.run(soft[:m])
        dt = time.perf_counter() - t0
        check(r["out"], sent, "reference")
        res["reference_1thread"] = dict(Msym_per_s=m / 2 / dt / 1e6, **{rt_key: m / 2 / dt / symrate})
    else:
        res["reference_1thread"] = None
    print(json.dumps(res))


if __name__ == "__main__":
    main()
