"""CPU: the drop-in boundary. The C-ABI library loads, exports every symbol include/b200dsp.h declares, validates
parameters like the reference modules do, and refuses to run without an H100 (there is no CPU fallback)."""
import ctypes
import os
import re

import pytest

from tests.common import ROOT


def test_library_exports_every_declared_symbol(built):
    from satdump_b200 import capi
    hdr = open(os.path.join(ROOT, "include", "b200dsp.h")).read()
    declared = sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 25
    L = ctypes.CDLL(capi.LIB_PATH)
    missing = [s for s in declared if not hasattr(L, s)]
    assert not missing, missing
    assert sorted(capi.SYMBOLS) == declared, "capi.SYMBOLS must list exactly the header's entry points"


def test_struct_layouts_match_header(built):
    """ctypes mirrors of the POD structs: sizes as the C compiler lays them out."""
    import subprocess
    import tempfile
    from satdump_b200 import capi
    src = '#include "b200dsp.h"\n#include <stdio.h>\nint main(){printf("%zu %zu %zu %zu\\n",sizeof(b200_demod_cfg),sizeof(b200_fec_cfg),sizeof(b200_demod_stats),sizeof(b200_fec_stats));return 0;}'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        sizes = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    assert sizes == [ctypes.sizeof(capi.DemodCfg), ctypes.sizeof(capi.FecCfg), ctypes.sizeof(capi.DemodStats), ctypes.sizeof(capi.FecStats)]


def test_parameter_validation_mirrors_reference_modules(built):
    from satdump_b200 import capi
    bad = [
        (dict(samplerate=6e6, symbolrate=233333, constellation="qpsk", rrc_alpha=0.5, final_samplerate=0), -1),  # resampler forced off
        (dict(samplerate=6e6, symbolrate=2333333, constellation="qpsk", rrc_alpha=0.5, rrc_taps=63), -1),
        (dict(samplerate=0, symbolrate=2333333, constellation="qpsk", rrc_alpha=0.5), -1),
        (dict(samplerate=30e6, symbolrate=25e6, constellation="oqpsk", rrc_alpha=0.5, final_samplerate=0), -1),  # OQPSK window is [1.6, 2.4]
        (dict(samplerate=6e6, symbolrate=2333333, constellation="qpsk", rrc_alpha=0.5, final_samplerate=30e6), -1),  # sps 12.9 after "resampling"
    ]
    for kw, code in bad:
        with pytest.raises(capi.B200Error) as e:
            capi.Demod(capi.demod_cfg(**kw))
        if isinstance(code, str):  # create() failures all surface as EINVAL in the binding; the text names the reason
            assert code in str(e.value), (kw, str(e.value))
        else:
            assert e.value.code == code, (kw, e.value.code)
    with pytest.raises(capi.B200Error):
        capi.Fec(capi.ccsds_cfg("8psk", 8192, 0.3, 20, 4))
    with pytest.raises(capi.B200Error):
        capi.Fec(capi.ccsds_cfg("qpsk", 8192, 0.3, 20, 5))  # 5 interleaved codewords do not fit 1024 bytes
    for cfg in (capi.simple_cfg("bpsk", 8192, 4, derand_start=-1), capi.ccsds_cfg("qpsk", 8192, 0.3, 20, 4, derand_start=-4, derand_after_rs=True)):
        with pytest.raises(capi.B200Error) as e:  # the derandomiser would start before the CADU
            capi.Fec(cfg)
        assert e.value.code == -1 and "derand_start" in str(e.value)


def test_no_cpu_fallback(built):
    """On a box without a GPU every create() must fail loudly with ENODEV — never compute on the host."""
    import torch
    from satdump_b200 import capi
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(capi.B200Error) as e:
        capi.Demod(capi.demod_cfg(6e6, 2333333, "qpsk", 0.5))
    assert e.value.code == -2 and "no cpu fallback" in str(e.value).lower()
    with pytest.raises(capi.B200Error) as e:
        capi.Fec(capi.metop_cfg())
    assert e.value.code == -2


def test_product_never_touches_the_oracle():
    """The product path (package + C sources + bench main arm) must not import / link the oracle."""
    for dp, _, fns in os.walk(os.path.join(ROOT, "satdump_b200")):
        for fn in fns:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".cpp")) or fn == "Makefile":
                txt = open(os.path.join(dp, fn), errors="ignore").read()
                assert "liboracle" not in txt and "libsatref" not in txt and "from oracle" not in txt and "import oracle" not in txt, fn


def test_bench_reference_arm_contract(built):
    """`bench.py --impl reference` (the reference's own threaded CPU pipeline from oracle/_ref, or the port where the reference is
    absent): exactly one JSON line on stdout with the contract's keys, same metric / unit / workload as the GPU arm."""
    import json
    import subprocess
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0", "--log2-samples", "22"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [x for x in r.stdout.splitlines() if x.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
              "config", "cpu_baseline", "e2e"):
        assert k in d, k
    sys.path.insert(0, ROOT)
    import bench
    assert d["impl"] == "reference" and d["unit"] == "MS/s" and d["config"]["workload"] == bench.WORKLOADS["c3"]["label"] and d["value"] > 0
    assert d["metric"] == bench.WORKLOADS["c3"]["metric"]
    assert d["e2e"] == {"value": d["value"], "unit": "MS/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and d["config"]["result_bytes_per_stream"] > 100 * 1024
    if cb["kind"] == "reference":  # both builds of the reference, median of >= 3 runs, per-stage single-thread rates (BASELINE.md 2.4)
        assert set(cb["variants"]) == {"generic_O2", "native_O3_fma"}
        for v in cb["variants"].values():
            assert len(v["one_stream_MSps_runs"]) >= 3 and v["stage_single_thread_MSps"]["fir"] > 0
