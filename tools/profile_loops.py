"""Diagnostic (not a test, not the bench): where the time of the demodulator's two loop stages goes in ONE synchronous step.

  python tools/profile_loops.py [config [log2 samples [Es/N0 dB]]]      (defaults: c3 29)

Runs a warm-up step, times three synchronous steps with CUDA events, then profiles one more step on its own with torch.profiler (CUDA
activities only) and prints per-kernel device times of the loop stages: k_costas and k_mm split into their main launch and the
repair launches (the 8-CTA grids), the fix-up / scan / compaction kernels, plus the demodulator's `repairs` and unconverged-junction
counters for that step (and where its repairs stopped: the checkpoint at which each met the stored run), the loop kernels' main-pass grids (segments / 128) and the card's name, power limit and SM clock.
For each main pass it also prints the bytes it moves (nseg x (L + W) input samples, its outputs) over its time, and its time as SM cycles
per sample (k_costas) or per symbol (k_mm) of one warp, at the SM clock read after the run.

  --lib PATH   time another build of libb200dsp.so (e.g. the parent commit's) instead of satdump_b200/csrc's: alternate two builds in
               one session to compare them
  --cycles     build the library with -DB200_LOOP_CYCLES into a temporary directory (unless --lib names one built so) and print where
               the main passes' cycles go: per warp, the row wait, the loop itself and the output path (clock64() totals of lane 0)
"""
import collections
import json
import math
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


def round_up16(x):
    return (int(math.ceil(x)) + 15) & ~15


def loop_geometry(cfg, n, nblk):
    """Segment count, L and the Costas / M&M warm-ups of a main pass of nblk CTAs, as the demodulator sets them (api_demod.cu) for a
    signal without a resampler, with the default clock_gain_mu."""
    nseg = nblk * SEG_THREADS
    L = round_up16(n / nseg)
    sps = cfg.samplerate / cfg.symbolrate
    wc = round_up16((72.0 if cfg.constellation == "8psk" else 24.0) / cfg.pll_bw)
    ref_sps = 2.5 if cfg.constellation == "bpsk" else 2.5714
    wm = round_up16((240.0 if cfg.constellation == "bpsk" else 87.5) * max(1.0, sps * sps / (ref_sps * ref_sps)) / 8.7e-3)
    return nseg, L, wc, wm, sps


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    flags = sys.argv[1:]
    if "--lib" in flags:
        capi.LIB_PATH = os.path.abspath(flags[flags.index("--lib") + 1])
        args.remove(flags[flags.index("--lib") + 1])
    cycles = "--cycles" in flags
    if cycles and "--lib" not in flags:
        out = os.path.join(tempfile.gettempdir(), "b200_loop_cycles")
        subprocess.run(["make", "-s", "-j8", "-C", os.path.join(os.path.dirname(bench.__file__), "satdump_b200", "csrc"), "cycles",
                        f"CYCLES_DIR={out}"], check=True, stdout=subprocess.DEVNULL)
        capi.LIB_PATH = os.path.join(out, "libb200dsp.so")
    wname = args[0] if len(args) > 0 else "c3"
    lg = int(args[1]) if len(args) > 1 else 29
    esn0 = float(args[2]) if len(args) > 2 else None
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
    if cycles:
        capi.loop_cycles()  # clear what the warm-up and the timed steps counted
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
    print(f"library {capi.LIB_PATH}")
    print(f"{'kernel':<18}{'launches':>9}{'ms':>10}")
    for k, (ms, cnt) in acc.items():
        if cnt:
            print(f"{k:<18}{cnt:>9}{ms:>10.3f}")
    lc = capi.loop_cycles() if cycles else None
    clock = card().get("clocks.sm", "")
    hz = float(clock.split()[0]) * 1e6 if clock[:1].isdigit() else None
    for k, unit in (("k_costas", "sample"), ("k_mm", "symbol")):
        if k not in grids or not acc[k][1]:
            continue
        nseg, L, wc, wm, sps = loop_geometry(cfg, n, grids[k])
        ms = acc[k][0]
        if k == "k_costas":
            steps, nbytes = L + wc, nseg * (L + wc) * 8 + n * 8  # per thread: samples; in: segments with warm-ups, out: the stream
        else:
            steps, nbytes = (L + wm) / sps, nseg * (L + wm) * 8 + int(n / sps) * 8  # in: segments with warm-ups, out: owned symbols
        per = f"{ms * 1e-3 * hz / steps:.0f} SM cycles per {unit} of one warp at {clock}" if hz else "SM clock not read"
        print(f"{k} main pass: nseg {nseg}, L {L}, W {wc if k == 'k_costas' else wm}: {nbytes / 1e9:.2f} GB in {ms:.3f} ms = "
              f"{nbytes / ms / 1e9:.2f} TB/s; {per}")
        if lc:
            c = lc[k]
            names = ("row wait", "Costas loop", "copy-out", "tail") if k == "k_costas" else ("row wait", "input fix-up", "symbol loop", "symbol copy-out")
            warps = max(1, c[4])
            tot = sum(c[:4])
            print(f"  clock64() per warp ({warps} warps, per {unit}: / {steps:.0f}): " + ", ".join(
                f"{nm} {v / warps:.0f} ({100 * v / max(1, tot):.1f} %, {v / warps / steps:.0f}/{unit})" for nm, v in zip(names, c[:4])))


if __name__ == "__main__":
    main()
