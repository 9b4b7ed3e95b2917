"""CPU: the prosody mix's host side - identities of its fp64 oracle, the weight and argument checks in Python and in C (no
CUDA call is made), and the ctypes mirror of the new entry points."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import ref_prosody_mix as PM
from conftest import ROOT


def rows(K, V, seed):
    return (np.random.default_rng(seed).standard_normal((K, V)) * 3).astype(np.float32)


def log_softmax(z):
    z = z.astype(np.float64)
    return z - z.max() - np.log(np.exp(z - z.max()).sum())


@pytest.mark.parametrize("V", [1024, 37])
def test_one_source_is_log_softmax(V):
    z = rows(1, V, V)
    z2 = np.concatenate([z, rows(1, V, V + 1)])
    # K = 1 with a positive weight is the one-weighted-source rule: the raw row
    assert np.array_equal(PM.mix_logprobs(z, [2.5]), z[0].astype(np.float64))
    # two copies of one source: the mixture is that source's log_softmax
    np.testing.assert_allclose(PM.mix_logprobs(np.concatenate([z, z]), [0.3, 0.7]), log_softmax(z[0]), atol=1e-12)
    assert PM.mix_logprobs(z2, [0.0, 1.0]).tolist() == z2[1].astype(np.float64).tolist()


def test_one_hot_weights_give_the_raw_row():
    z = rows(3, 64, 1)
    z[1, 5] = np.nan
    z[1, 9] = np.inf
    for k in range(3):
        w = np.zeros(3)
        w[k] = 0.25
        got = PM.mix_logprobs(z, w)
        assert np.array_equal(got, z[k].astype(np.float64), equal_nan=True)


def test_weights_are_scale_invariant():
    z = rows(3, 200, 2)
    a = PM.mix_logprobs(z, [0.2, 0.3, 0.5])
    np.testing.assert_allclose(PM.mix_logprobs(z, [2.0, 3.0, 5.0]), a, rtol=0, atol=1e-7)     # fp32 weights
    np.testing.assert_allclose(np.exp(a).sum(), 1.0, atol=1e-12)
    # and the mixture sits between its sources: log-sum-exp of log w + log_softmax
    want = np.logaddexp.reduce(np.log([0.2, 0.3, 0.5])[:, None] + np.stack([log_softmax(r) for r in z]), axis=0)
    np.testing.assert_allclose(a, want, atol=1e-7)


def test_non_finite_rules():
    V = 8
    z = np.zeros((2, V), np.float32)
    z[0] = [np.nan, -np.inf, 1, 2, np.inf, 0, np.inf, 3]         # +inf: all of source 0's mass on index 4
    z[1] = [np.nan] * V                                           # no candidate: contributes nothing
    l = PM.mix_logprobs(z, [1, 1])
    assert l[4] == np.log(0.5) and np.all(l[np.arange(V) != 4] == -np.inf)
    z[1] = -np.inf
    z[0] = np.nan
    assert np.all(PM.mix_logprobs(z, [1, 3]) == -np.inf)
    assert PM.mix_pick(z, [1, 3]) == (0, np.inf)
    # NaN / -inf have no mass; the other tokens renormalise within their source
    z = np.array([[np.nan, 0.0, 0.0, -np.inf], [0.0, 0.0, 0.0, 0.0]], np.float32)
    np.testing.assert_allclose(np.exp(PM.mix_logprobs(z, [1, 1])), [0.125, 0.375, 0.375, 0.125], atol=1e-15)


def test_mix_pick_follows_the_sampler_rules():
    z = rows(2, 300, 3)
    l = PM.mix_logprobs(z, [0.4, 0.6])
    pick, gap = PM.mix_pick(z, [0.4, 0.6])
    assert pick == int(np.argmax(l)) and gap > 0
    from oracle import ref_sampling as RS
    smp = (0.8, 20, 0.9, 12345)
    pick, _ = PM.mix_pick(z, [0.4, 0.6], 7, smp, 99)
    assert pick == RS.sample_row(l.astype(np.float32), 7, *smp, 99)[0]
    assert PM.mix_pick(z, [0.4, 0.6], 7, (0.0, 0, 1.0, 1), 99)[0] == int(np.argmax(l))


# ------------------------------------------------------------------------------ argument validation
def test_mix_weights_validation():
    from megatts2_b200 import _lib as L
    from megatts2_b200.sampling import mix_weights
    w = mix_weights([1, 3], 2, 3)
    assert w.dtype == torch.float32 and w.shape == (3, 2) and w.is_contiguous() and w[2].tolist() == [1.0, 3.0]
    assert mix_weights(torch.tensor([[0.5, 0.0], [0.0, 2.0]]), 2, 2).tolist() == [[0.5, 0.0], [0.0, 2.0]]
    assert mix_weights(np.ones(8), 8, 1).shape == (1, 8)
    bad = [([1.0, -0.1], 2, 1), ([1.0, float("nan")], 2, 1), ([1.0, float("inf")], 2, 1), ([0.0, 0.0], 2, 1),
           ([1.0, 2.0, 3.0], 2, 1), ([[1.0, 1.0]], 2, 2), ([1e-46, 0.0], 2, 1), ([3e38, 3e38], 2, 1),
           ([1.0] * 9, 9, 1), ([], 0, 1), ([True, False], 2, 1), ("ab", 2, 1), ([[1.0, 0.0], [0.0, 0.0]], 2, 2)]
    for weights, K, B in bad:
        with pytest.raises(L.MttsError):
            mix_weights(weights, K, B)


def test_python_entry_points_reject_malformed_sources():
    """infer_mix / synthesize check their arguments on the host before any device call."""
    from megatts2_b200 import _lib as L
    from megatts2_b200.models.megatts2 import MegaPLM, Megatts
    plm = MegaPLM(n_layers=1, n_heads=2, vq_dim=8, tc_latent_dim=8, vq_bins=16).eval()
    with pytest.raises(L.MttsError):
        plm.infer_mix(torch.zeros(1, 2, 8), [1.0])                # a tensor, not a list
    with pytest.raises(L.MttsError):
        plm.infer_mix([], [1.0])
    with pytest.raises(L.MttsError):
        plm.infer_mix([torch.zeros(1, 2, 8)], [1.0])              # CPU tensors: no fallback
    tts = Megatts.__new__(Megatts)
    phone = torch.zeros(2, 3, dtype=torch.int64)
    for kw in (dict(prosody_mels=None, prosody_weights=[1.0]), dict(prosody_mels=[], prosody_weights=[1.0]),
               dict(prosody_mels=torch.zeros(2, 4, 80), prosody_weights=[1.0, 1.0]),
               dict(prosody_mels=[object()], prosody_weights=None)):
        with pytest.raises(L.MttsError):
            tts._check_prosody(phone, kw["prosody_mels"], kw["prosody_weights"], False)
    with pytest.raises(L.MttsError, match="causal"):
        tts._check_prosody(phone, [torch.zeros(2, 4, 80)], [1.0, 1.0], True)
    with pytest.raises(L.MttsError, match="synthesize_many"):
        Megatts.synthesize_many(tts, [], prosody_mels=[torch.zeros(1, 4, 80)], prosody_weights=[1, 1])


def test_c_side_rejects_bad_mix_arguments():
    """The C entry points validate before they enqueue anything (so no device is needed to see the errors)."""
    from megatts2_b200 import _lib as L
    lib = L.lib()
    dummy = C.c_void_p(256)                    # never dereferenced: every call below fails its checks first
    assert lib.mtts_mix_logprob_rows_f32(dummy, 1024, 1024, 9, 4, dummy, dummy, 1024, None) == -2
    assert "K = 9" in lib.mtts_last_error().decode()
    assert lib.mtts_mix_logprob_rows_f32(dummy, 4097, 4097, 2, 4, dummy, dummy, 4097, None) == -2
    assert "4096" in lib.mtts_last_error().decode()
    assert lib.mtts_mix_logprob_rows_f32(dummy, 1024, 1024, 0, 4, dummy, dummy, 1024, None) == -1
    assert lib.mtts_mix_logprob_rows_f32(None, 1024, 1024, 2, 4, dummy, dummy, 1024, None) == -1
    assert lib.mtts_mix_logprob_rows_f32(dummy, 1024, 1024, 2, 0, dummy, dummy, 1024, None) == 0     # nothing to do
    assert lib.mtts_plm_infer_mix_f32(None, 2, None, 0, 0, 1, 1, None, None, None, None, None, 0, None) == -1
    assert lib.mtts_plm_infer_mix_range_f32(None, 2, None, 0, 0, 1, 1, None, 0, 1, None, None, None, None, None, 0,
                                            None) == -1
    # a PLM descriptor whose pointers are never followed: the K / V / weights checks come first
    layer = L.EncoderLayer()
    plm = L.PLM()
    plm.enc.layers = C.pointer(layer)
    plm.enc.d_model, plm.tc_dim, plm.vq_dim, plm.vq_bins = 16, 8, 8, 1024
    plm.pc_embedding = plm.w_predict = plm.pe = 256

    def mix(K, V=1024, weights=dummy, s=None):
        plm.vq_bins = V
        return lib.mtts_plm_infer_mix_f32(C.byref(plm), K, dummy, 0, 8, 1, 1, weights, dummy, None, s, dummy, 1 << 30,
                                          None)
    assert mix(9) == -2 and "K = 9" in lib.mtts_last_error().decode()
    assert mix(2, V=5000) == -2
    assert mix(2, weights=None) == -1
    bad = L.Sampling(-1.0, 0, 1.0, 0, 256, 256)
    assert mix(2, s=C.byref(bad)) == -1 and "temperature" in lib.mtts_last_error().decode()
    assert lib.mtts_plm_infer_mix_range_f32(C.byref(plm), 2, dummy, 0, 8, 1, 4, dummy, 3, 2, dummy, dummy, None, None,
                                            dummy, 1 << 30, None) == -1                          # t0 > t1
    assert lib.mtts_plm_infer_mix_workspace_bytes(C.byref(plm), 2, 4, 8) > lib.mtts_plm_infer_workspace_bytes(
        C.byref(plm), 4, 8)


def test_ctypes_signatures_match_the_header():
    """Argument counts of the new entry points in _lib.SIGNATURES against their prototypes in the C header."""
    import os
    from megatts2_b200 import _lib as L
    src = open(os.path.join(ROOT, "include", "megatts2_b200.h")).read()
    for name in ("mtts_mix_logprob_rows_f32", "mtts_plm_infer_mix_workspace_bytes", "mtts_plm_infer_mix_f32",
                 "mtts_plm_infer_mix_range_f32"):
        m = re.search(r"\b" + name + r"\(([^)]*)\)", src)
        assert m, name
        n_args = len([a for a in m.group(1).split(",") if a.strip()])
        assert len(L.SIGNATURES[name][1]) == n_args, name
        assert L.SIGNATURES[name][0] is (C.c_int64 if name.endswith("_bytes") else C.c_int), name
