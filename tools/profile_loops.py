"""Diagnostic (not a test, not the bench): where the time of the demodulator's two loop stages goes in ONE synchronous step.

  python tools/profile_loops.py [config [log2 samples [Es/N0 dB]]]      (defaults: c3 29)

Runs a warm-up step, times three synchronous steps with CUDA events, then profiles one more step on its own with torch.profiler (CUDA
activities only) and prints per-kernel device times of the loop stages: k_costas and k_mm split into their main launch and the
repair launches (the 8-CTA grids), the fix-up / scan / compaction kernels, plus the demodulator's `repairs` and unconverged-junction
counters for that step (and where its repairs stopped: the checkpoint at which each met the stored run), the loop kernels' main-pass grids (segments / 128) and the card's name, power limit and SM clock.
"""
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from satdump_b200 import capi  # noqa: E402

KERNELS = ("k_costas", "k_costas_fix", "k_pll", "k_mm", "k_mm_scan", "k_mm_compact", "k_snr_m2m4")
LOOP_KERNELS = ("k_costas", "k_pll", "k_mm")  # launched on nblk CTAs for the main pass and on 8 CTAs per repair round
SEG_THREADS = 128  # segments per CTA of the loop kernels (satdump_b200/csrc/demod.cuh)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), (v.strip() for v in out.strip().split(","))))
    except (OSError, subprocess.SubprocessError):
        return {}


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    wname = sys.argv[1] if len(sys.argv) > 1 else "c3"
    lg = int(sys.argv[2]) if len(sys.argv) > 2 else 29
    esn0 = float(sys.argv[3]) if len(sys.argv) > 3 else None
    w = bench.WORKLOADS[wname]
    assert w["kind"] == "chain", "the loop stages are profiled through a chain workload"
    cfg, raw, _ = bench.make_workload(w, lg, 0, "cuda", esn0)
    n = bench.nsamples_of(raw, cfg)
    pipe = bench.ChainPipe(capi, cfg, n, 0)

    def step():
        pipe.reset()
        pipe.push_device(raw.data_ptr(), n)
        pipe.ch.sync()

    step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    step_ms = []
    for _ in range(3):
        t0.record()
        step()
        t1.record()
        torch.cuda.synchronize()
        step_ms.append(t0.elapsed_time(t1))
    timing = pipe.timing()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    dstats = pipe.stats()["demod"]  # reset() clears the counters: these are the profiled step's own
    merge_hist = pipe.ch.stats()[0]["repair_merge_hist"]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    acc = collections.OrderedDict((k, [0.0, 0]) for k in ("k_costas", "k_costas repair", "k_costas_fix", "k_pll", "k_pll repair", "k_mm", "k_mm repair",
                                                           "k_mm_scan", "k_mm_compact", "k_snr_m2m4"))
    grids = {}
    for ev in trace.get("traceEvents", []):
        if ev.get("cat") != "kernel":
            continue
        m = re.search(r"\b(k_\w+)", ev.get("name", ""))
        if not m or m.group(1) not in KERNELS:
            continue
        k = m.group(1)
        grid = ev.get("args", {}).get("grid", [0])[0]
        if k in LOOP_KERNELS:
            if grid == 8:
                k += " repair"
            else:
                grids[k] = grid
        acc[k][0] += ev["dur"] / 1000.0
        acc[k][1] += 1
    print(f"config {wname}, 2^{lg} samples, card {card()}")
    print(f"synchronous step: {' '.join(f'{x:.2f}' for x in step_ms)} ms (CUDA events), stage_ms {json.dumps(timing)}")
    print(f"demodulator counters of the profiled step: {dstats}; main-pass grids (CTAs of {SEG_THREADS} segments): {grids}")
    buckets = ["whole segment", "1", "2", "3-4", "5-8", "9-16", "17-32", ">32"]
    print(f"repairs by the {capi.CKPT}-sample checkpoint at which they met the stored run and stopped: {dict(zip(buckets, merge_hist))}")
    print(f"{'kernel':<18}{'launches':>9}{'ms':>10}")
    for k, (ms, cnt) in acc.items():
        if cnt:
            print(f"{k:<18}{cnt:>9}{ms:>10.3f}")


if __name__ == "__main__":
    main()
