"""CPU: the checkers of ccsds_ldpc_decoder (rate 7/8 C2 code). The parity-check matrix of satdump_b200/csrc/ldpc_c2_table.inc is the
reference's; the C restatement (oracle/ldpc_port.c) equals the reference's own decoder, correlator and module loop bit for bit (directly
against oracle/_ref, or through the digests of tests/golden/ldpc_pins.json where it is absent); synthesised codewords satisfy H c = 0
and decode to the transmitted frames; and the decoder's configuration refuses what is not built, by name."""
import functools
import hashlib
import os

import numpy as np
import pytest

from oracle import ldpc as O
from satdump_b200 import synth
from tests.common import ROOT, load_pins

PINS = os.path.join(ROOT, "tests", "golden", "ldpc_pins.json")
# decoder alone: random LLRs (sigma) at 1, 10 and 50 iterations; module loop: soft streams (constellation, sigma, rotation, Q late, edit)
CASES = {f"dec_s{s}_it{it}": (s, it) for s in (20, 45, 90) for it in (1, 10, 50)}
CASES.update({"loop_bpsk": ("bpsk", 22.0, 0, False, None), "loop_qpsk_rot1": ("qpsk", 25.0, 1, False, None),
              "loop_oqpsk_rot3_late": ("oqpsk", 22.0, 3, True, None), "loop_qpsk_edit": ("qpsk", 18.0, 0, False, "edit"),
              "loop_bpsk_noise": ("bpsk", 15.0, 0, False, "noise"), "loop_oqpsk_inner_8272": ("oqpsk", 18.0, 1, False, "inner8272"),
              "loop_qpsk_inner_14304": ("qpsk", 18.0, 0, False, "inner14304")})


@pytest.fixture(scope="module")
def libs(built):
    if not O.available("port"):
        import __graft_entry__ as g
        g.build()
    return True


def _h(*arrays):
    m = hashlib.sha256()
    for a in arrays:
        m.update(np.ascontiguousarray(a).tobytes())
    return m.hexdigest()


def decode_inputs(name):
    sigma, it = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    bits = rng.integers(0, 2, (4, 8158))
    return np.clip(np.round((bits * 2.0 - 1) * 40 + rng.normal(0, sigma, bits.shape)), -128, 127).astype(np.int8), it


def digest_decode(name, impl):
    cws, it = decode_inputs(name)
    f = O.Fec(O.ldpc_cfg("qpsk", it), impl)
    outs = [f.decode(cw) for cw in cws]
    return _h(np.stack([o[0] for o in outs]), np.array([o[1] for o in outs], np.int64))


def stream_input(name):
    cons, sigma, rot, late, edit = CASES[name]
    seed = sum(map(ord, name))
    rng = np.random.default_rng(seed)
    if edit and edit.startswith("inner"):
        info, _ = synth.ldpc_inner_frames(5, int(edit[5:]), 0x352EF853, seed)
        tx, _, _ = synth.ldpc_frames(5, seed, info=info)
    else:
        tx, _, _ = synth.ldpc_frames(5, seed)
    bits = np.concatenate([rng.integers(0, 2, 1234 * 2, dtype=np.uint8), tx.reshape(-1), rng.integers(0, 2, 999 * 2, dtype=np.uint8)])
    soft = synth.ldpc_soft(bits, cons, sigma=sigma, rot=rot, q_late=late, seed=seed)
    if edit == "edit":
        soft = np.concatenate([soft[:2468 + 2 * 8192 + 77], np.full(41, 3, np.int8), soft[2468 + 2 * 8192 + 77:2468 + 4 * 8192],
                               soft[2468 + 4 * 8192 + 500:]])
    elif edit == "noise":
        noise = np.clip(np.round(rng.normal(0, 40, 2 * 8192 + 555)), -127, 127).astype(np.int8)
        soft = np.concatenate([noise, soft, noise])
    return soft


def run_stream(name, impl):
    edit = CASES[name][4]
    inner = int(edit[5:]) if edit and edit.startswith("inner") else 0
    return O.Fec(O.ldpc_cfg(CASES[name][0], internal_cadu_size=inner, internal_asm=0x352EF853), impl).run(stream_input(name))


def digest_stream(name, impl):
    r = run_stream(name, impl)
    return _h(r["cadu"], r["recs"])


def digest_matrix(impl):
    return _h(O.matrix(impl).astype(np.int32))


pins = functools.partial(load_pins, PINS)


def test_table_reproduces_the_reference_matrix(libs):
    """H from ldpc_c2_table.inc (synth and the restatement) = make_r78_code()'s matrix, rows row-block-major, columns ascending."""
    cols = synth.ldpc_c2_cols().astype(np.int32)
    assert np.array_equal(O.matrix("port"), cols)
    if O.available("ref"):
        assert np.array_equal(O.matrix("ref"), cols)
    assert digest_matrix("port") == pins()["matrix"]
    H = synth.ldpc_c2_h()
    assert H.shape == (1022, 8176) and (H.sum(1) == 32).all() and (H.sum(0) == 4).all()


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("dec_")])
def test_restated_decoder_bit_exact(libs, name):
    if O.available("ref"):
        cws, it = decode_inputs(name)
        r, p = O.Fec(O.ldpc_cfg("qpsk", it), "ref"), O.Fec(O.ldpc_cfg("qpsk", it), "port")
        for cw in cws:
            a, b = r.decode(cw), p.decode(cw)
            assert np.array_equal(a[0], b[0]) and a[1] == b[1]
    assert digest_decode(name, "port") == pins()[name]


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("loop_")])
def test_restated_module_loop_bit_exact(libs, name):
    """Correlator decisions (offset, pos, correlator_corr bits, phase, swap), ldpc_corr and the CADUs of the module loop."""
    p = run_stream(name, "port")
    assert p["cadu"].shape[0] >= (2 if "inner" in name else 3)
    if O.available("ref"):
        r = run_stream(name, "ref")
        assert np.array_equal(r["recs"], p["recs"]) and np.array_equal(r["cadu"], p["cadu"])
    assert digest_stream(name, "port") == pins()[name]


def test_synthesised_codewords_decode_to_the_transmitted_frames(libs):
    tx, cw, clear = synth.ldpc_frames(4, 77)
    assert not ((cw.astype(np.int64) @ synth.ldpc_c2_h().T.astype(np.int64)) % 2).any()
    assert not cw[:, :18].any() and tx.shape == (4, 8192)
    soft = synth.ldpc_soft(np.concatenate([np.zeros(64, np.uint8), tx.reshape(-1)]), "qpsk", sigma=20.0, seed=1)
    got = O.Fec(O.ldpc_cfg("qpsk")).run(soft)
    assert np.array_equal(got["cadu"], clear)
    assert got["recs"][0, 1] == 64 and (got["recs"][1:, 1] == 0).all()


@pytest.mark.parametrize("kw,code,word", [(dict(ldpc_rate="1/2", ldpc_block_size=1024), -6, "AR4JA"), (dict(ldpc_rate="2/3"), -6, "AR4JA"),
                                          (dict(ldpc_rate="4/5", ldpc_block_size=16384), -6, "AR4JA"), (dict(ldpc2=True), -6, "ldpc2"),
                                          (dict(internal_stream=True, internal_cadu_size=8276), -6, "padding"),
                                          (dict(internal_stream=True, internal_cadu_size=32), -1, "internal_cadu_size"),
                                          (dict(constellation="8psk"), -6, "8PSK"), (dict(constellation="bpsk_90"), -1, "constellation"),
                                          (dict(ldpc_iterations=-1), -1, "ldpc_iterations")])
def test_ldpc_cfg_rejections_name_the_option(built, kw, code, word):
    """Refused before the device is looked at, so this holds on a machine without a GPU."""
    import ctypes
    from satdump_b200 import capi
    kw = dict(kw)
    cons = kw.pop("constellation", "qpsk")
    assert not capi.lib().b200_fec_create(ctypes.byref(capi.ldpc_cfg(cons, **kw)))
    assert word in capi.last_error()
    assert ("not built" in capi.last_error()) == (code == -6)
