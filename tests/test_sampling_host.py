"""CPU: the opt-in PLM sampler's host side - the oracle's Philox against the Random123 known-answer vectors, the oracle's
filters on hand-made rows, the ``Sampling`` parameter checks in Python and in C (no CUDA call is made), and the ctypes
mirror of ``mtts_sampling``."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle import ref_sampling as RS

KAT = [  # (counter, key) -> output, Random123 kat_vectors for philox4x32_10
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_oracle_philox_known_answers(ctr, key, want):
    assert tuple(int(w) for w in RS.philox4x32_10(np.array(ctr), np.array(key))) == want


def test_oracle_word_layout():
    """Token i reads word i & 3 of the Philox block with counter (i >> 2, t, key_lo, key_hi) and key (seed_lo, seed_hi)."""
    seed, key, t = 0x0123456789ABCDEF, 0xFEDCBA9876543210, 77
    idx = np.arange(12)
    w = RS.words(seed, key, t, idx)
    for i in idx:
        blk = RS.philox4x32_10(np.array([i >> 2, t, key & 0xFFFFFFFF, key >> 32]), np.array([seed & 0xFFFFFFFF, seed >> 32]))
        assert int(w[i]) == int(blk[i & 3])


def test_oracle_gumbel_noise_is_finite_at_the_ends():
    g = RS.gumbel(np.array([0, 255, 256, 2 ** 31, 2 ** 32 - 257, 2 ** 32 - 1], dtype=np.uint64))
    assert np.isfinite(g).all() and g[0] == g[1] and (np.diff(g)[1:] > 0).all()       # the low 8 bits are dropped
    u_top = (2 ** 24 - 1 + 0.5) * 2.0 ** -24
    assert g[-1] == pytest.approx(-math.log(-math.log1p(-(1 - u_top))), rel=1e-12)


def test_oracle_filters_on_hand_made_rows():
    z = np.array([1.0, 3.0, 3.0, -0.0, 0.0, np.nan, -np.inf, 2.0], dtype=np.float32)
    kept, _ = RS.kept_set(RS.tempered(z, 1.0), 0, 1.0)
    assert kept.tolist() == [1, 2, 7, 0, 3, 4]                         # value desc, index asc; -0 ties with +0; no NaN/-inf
    assert RS.kept_set(RS.tempered(z, 1.0), 2, 1.0)[0].tolist() == [1, 2]
    assert RS.kept_set(RS.tempered(z, 1.0), 8, 1.0)[0].tolist() == [1, 2, 7, 0, 3, 4]   # k >= V: off
    assert RS.kept_set(RS.tempered(z, 1.0), 0, 1e-9)[0].tolist() == [1]
    flat = np.zeros(8, dtype=np.float32)
    assert RS.kept_set(RS.tempered(flat, 1.0), 0, 0.5)[0].tolist() == [0, 1, 2, 3]     # cumulative mass 4/8 >= 0.5
    assert RS.kept_set(RS.tempered(flat, 1.0), 0, 0.51)[0].tolist() == [0, 1, 2, 3, 4]
    p = RS.target_distribution(flat, 1.0, 3, 1.0)
    assert np.allclose(p, [1 / 3] * 3 + [0] * 5)
    # edge rows
    assert RS.sample_row(np.array([0, np.inf, 1, np.inf], dtype=np.float32), 0, 1.0, 0, 0.9, 1, 2)[0] == 1
    assert RS.sample_row(np.array([np.nan, -np.inf, np.nan], dtype=np.float32), 0, 1.0, 0, 1.0, 1, 2)[0] == 0
    assert RS.sample_row(np.array([np.nan, 5, 7, 7], dtype=np.float32), 3, 0.0, 0, 1.0, 1, 2)[0] == 2     # greedy
    assert RS.sample_row(np.array([np.nan, 5, 7, 7], dtype=np.float32), 3, 2.0, 1, 1.0, 1, 2)[0] == 2
    assert RS.greedy(np.array([np.nan, -np.inf], dtype=np.float32)) == 0


@pytest.mark.parametrize("kw", [dict(temperature=-1.0), dict(temperature=float("nan")), dict(temperature=float("inf")),
                                dict(temperature=1e39), dict(temperature=True), dict(temperature="1"),
                                dict(top_k=-1), dict(top_k=1.5), dict(top_k=True), dict(top_k=2 ** 31),
                                dict(top_p=0.0), dict(top_p=1.1), dict(top_p=float("nan")), dict(top_p=1e-50),
                                dict(top_p=-0.5), dict(seed=-1), dict(seed=2 ** 64), dict(seed=1.0)])
def test_sampling_rejects_out_of_range_fields(kw):
    from megatts2_b200 import _lib as L
    from megatts2_b200.sampling import Sampling
    with pytest.raises(L.MttsError):
        Sampling(**kw)


def test_sampling_fields_and_graph_key():
    import torch
    from megatts2_b200.sampling import Sampling, row_keys
    s = Sampling(temperature=0.7, top_k=np.int64(20), top_p=0.9, seed=2 ** 64 - 1)
    assert s.top_k == 20 and isinstance(s.top_k, int) and s == Sampling(0.7, 20, 0.9, 2 ** 64 - 1)
    assert s.graph_key() == (C.c_float(0.7).value, 20, C.c_float(0.9).value)
    assert Sampling().graph_key() == (1.0, 0, 1.0) and Sampling(temperature=0).temperature == 0.0
    with pytest.raises(Exception):
        s.seed = 3                                                         # frozen
    assert row_keys(None, 3, "cpu").tolist() == [0, 1, 2]
    assert row_keys([5, 5], 2, "cpu").dtype == torch.int64
    from megatts2_b200 import _lib as L
    with pytest.raises(L.MttsError):
        row_keys([1, 2, 3], 2, "cpu")
    with pytest.raises(L.MttsError):
        row_keys(torch.tensor([0.5, 1.0]), 2, "cpu")


def test_c_side_rejects_bad_sampling_parameters():
    """The C entry points validate before they enqueue anything (so no device is needed to see the errors)."""
    from megatts2_b200 import _lib as L
    lib = L.lib()
    dummy = C.c_void_p(256)                    # never dereferenced: every call below fails its checks first

    def call(V=1024, **kw):
        f = dict(temperature=1.0, top_k=0, top_p=1.0, reserved=0, seed=dummy.value, keys=dummy.value)
        f.update(kw)
        s = L.Sampling(f["temperature"], f["top_k"], f["top_p"], f["reserved"], f["seed"], f["keys"])
        rc = lib.mtts_sample_rows_f32(dummy, 1024, V, 4, 0, C.byref(s), dummy, 1, None)
        return rc, lib.mtts_last_error().decode()

    for kw, msg in ((dict(temperature=-1.0), "temperature"), (dict(temperature=float("inf")), "temperature"),
                    (dict(temperature=float("nan")), "temperature"), (dict(top_k=-3), "top_k"),
                    (dict(top_p=0.0), "top_p"), (dict(top_p=1.5), "top_p"), (dict(top_p=float("nan")), "top_p"),
                    (dict(seed=None), "seed"), (dict(keys=None), "keys"), (dict(reserved=1), "reserved")):
        rc, err = call(**kw)
        assert rc == -1 and msg in err, (kw, err)
    rc, err = call(V=4097)
    assert rc == -2 and "4096" in err
    assert lib.mtts_sample_rows_f32(dummy, 1024, 1024, 4, 0, None, dummy, 1, None) == -1
    assert lib.mtts_plm_infer_sample_f32(None, None, 0, 0, 1, 1, None, None, None, None, 0, None) == -1
    assert lib.mtts_plm_decode_causal_sample_f32(None, None, 0, 0, 1, 1, None, None, None, None, 0, None) == -1


def test_sampling_struct_matches_the_c_header(tmp_path):
    from megatts2_b200 import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "megatts2_b200.h"', "int main(void) {",
             '  printf("sizeof %zu\\n", sizeof(mtts_sampling));']
    lines += [f'  printf("{f} %zu\\n", offsetof(mtts_sampling, {f}));' for f, _ in L.Sampling._fields_]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text("\n".join(lines))
    subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(re.match(r"(\w+) (\d+)", ln).groups() for ln in
               subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(got["sizeof"]) == C.sizeof(L.Sampling)
    for f, _ in L.Sampling._fields_:
        assert int(got[f]) == getattr(L.Sampling, f).offset, f
