"""CPU: the duration mix's host side - identities of its oracle (tests/ref_duration_mix.py), the argument checks in Python
and in C (no CUDA call is made), the entry points MegaADM.infer_mix calls, and the ctypes mirror of the new entries."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import ref_duration_mix as DM
from conftest import ROOT
from oracle import ref_megatts2 as R
from oracle import weights
from test_plm_dispatch_host import M_ADM, P, WS_OK, _adm, _latent, lib  # noqa: F401  (lib: the recorder fixture)


def gen(seed):
    return torch.Generator().manual_seed(seed)


def sources(K, B, T, seed):
    return [torch.randn(B, T, 512, generator=gen(seed + k)).abs() for k in range(K)]


# ------------------------------------------------------------------------------ oracle identities
def test_mix_readout_rules():
    y = torch.tensor([-0.0, float("nan"), 2.5, float("inf")], dtype=torch.float64)
    r = DM.mix_readout(y, [3.0, 0.0, 0.0, 0.0])                # one positive weight: that y, -0 kept
    assert r.item() == 0.0 and torch.signbit(r)
    assert DM.mix_readout(y, [0.0, 0.0, 1.0, 0.0]).item() == 2.5   # NaN and inf sources skipped at weight 0
    assert DM.mix_readout(y, [0.0, 0.0, 0.0, 0.0]).item() == 0.0   # the empty sum
    got = DM.mix_readout(torch.tensor([1.0, 4.0], dtype=torch.float64), [0.25, 0.75])
    assert got.item() == 3.25


def test_one_hot_and_one_source_equal_adm_infer(weights_cpu):
    """One positive weight decodes exactly what R.adm_infer decodes from that source; K = 1 is R.adm_infer."""
    sd, cfg = R.SD(weights_cpu("adm")), weights.ADM_CFG
    K, B, T = 3, 2, 5
    tcs = sources(K, B, T, 10)
    with torch.no_grad():
        refs = [R.adm_infer(sd, tc, cfg, return_raw=True) for tc in tcs]
        for k in range(K):
            w = np.zeros((B, K), np.float32)
            w[:, k] = 0.375
            dur, raw, raw_src = DM.adm_infer_mix(sd, tcs, cfg, w, return_raw=True)
            assert torch.equal(dur, refs[k][0]) and torch.equal(raw, refs[k][1]), k
            assert torch.equal(raw_src[k], refs[k][1][..., 0]), k
        dur, raw = DM.adm_infer_mix(sd, tcs[:1], cfg, np.full((B, 1), 2.0, np.float32), return_raw=True)[:2]
        assert torch.equal(dur, refs[0][0]) and torch.equal(raw, refs[0][1])


def test_power_of_two_scaling_changes_nothing(weights_cpu):
    sd, cfg = R.SD(weights_cpu("adm")), weights.ADM_CFG
    K, B, T = 2, 2, 4
    tcs = sources(K, B, T, 20)
    w = np.array([[0.3, 0.7], [0.55, 0.2]], np.float32)
    with torch.no_grad():
        a = DM.adm_infer_mix(sd, tcs, cfg, w, return_raw=True)
        b = DM.adm_infer_mix(sd, tcs, cfg, w * np.float32(2.0 ** 7), return_raw=True)
        c = DM.adm_infer_mix(sd, tcs, cfg, w * np.float32(2.0 ** -5), return_raw=True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    for x, y in zip(a, c):
        assert torch.equal(x, y)
    # the mix really lies between the sources: not equal to either one-hot decode
    assert not torch.equal(a[1][..., 0], a[2][0]) and not torch.equal(a[1][..., 0], a[2][1])


def test_fp64_oracle_is_close_to_fp32(weights_cpu):
    """The fp64 restatement and the fp32 one agree to fp32 rounding: what the GPU tests compare against is the model."""
    sd32, cfg = R.SD(weights_cpu("adm")), weights.ADM_CFG
    sd = DM.sd64(weights_cpu("adm"))
    tcs = sources(2, 2, 4, 30)
    w = np.array([[0.4, 0.6], [1.0, 0.0]], np.float32)
    with torch.no_grad():
        raw32 = DM.adm_infer_mix(sd32, tcs, cfg, w, return_raw=True)[1]
        raw64 = DM.adm_infer_mix(sd, [t.double() for t in tcs], cfg, w, return_raw=True)[1]
    assert raw64.dtype == torch.float64
    assert (raw32.double() - raw64).abs().max().item() <= 1e-3 * max(1.0, raw64.abs().max().item())


# ------------------------------------------------------------------------------ argument validation
def test_python_entry_points_reject_malformed_arguments():
    """infer_mix / synthesize check their arguments on the host before any device call."""
    from megatts2_b200 import _lib as L
    from megatts2_b200.models.megatts2 import MegaADM, Megatts
    adm = MegaADM(n_layers=1, n_heads=2, emb_dim=8, tc_latent_dim=8, tc_emb_dim=8).eval()
    for bad in (torch.zeros(1, 2, 8), [], [torch.zeros(1, 2, 8)]):         # a tensor; empty; CPU tensors (no fallback)
        with pytest.raises(L.MttsError):
            adm.infer_mix(bad, [1.0])
    tts = Megatts.__new__(Megatts)
    phone = torch.zeros(2, 3, dtype=torch.int64)
    with pytest.raises(L.MttsError, match="duration_weights without prosody_mels"):
        tts._check_prosody(phone, None, None, False, [1.0])


def test_synthesize_rejects_malformed_duration_weights(monkeypatch):
    """Wrong K and malformed weights raise in _check_prosody, named as the duration mix.  (The prompts are checked with
    ops._dev, replaced here so that CPU tensors stand in for device ones.)"""
    from megatts2_b200 import _lib as L
    from megatts2_b200 import ops
    from megatts2_b200.models.megatts2 import Megatts
    monkeypatch.setattr(ops, "_dev", lambda t, dtype=torch.float32, name="tensor": t)
    tts = Megatts.__new__(Megatts)
    tts.generator = type("G", (), {"mrte": type("M", (), {"mel_bins": 80})()})()
    phone = torch.zeros(2, 3, dtype=torch.int64)
    pros = [torch.zeros(2, 4, 80)]
    tts._check_prosody(phone, pros, [1.0, 1.0], False, [0.5, 0.5])       # well-formed: no error
    tts._check_prosody(phone, pros, [1.0, 1.0], False, torch.tensor([[1.0, 0.0], [0.0, 2.0]]))
    for dw in ([1.0], [1.0, 1.0, 1.0], [1.0, -1.0], [0.0, 0.0], [1.0, float("nan")], [1.0, float("inf")],
               torch.ones(3, 2), [[1.0, 1.0], [0.0, 0.0]], "ab"):
        with pytest.raises(L.MttsError, match="duration mix"):
            tts._check_prosody(phone, pros, [1.0, 1.0], False, dw)
    with pytest.raises(L.MttsError, match="causal"):
        tts._check_prosody(phone, pros, [1.0, 1.0], True, [1.0, 1.0])


def test_c_side_rejects_bad_mix_arguments():
    """The C entry points validate before they enqueue anything (so no device is needed to see the errors)."""
    from megatts2_b200 import _lib as L
    lib_ = L.lib()
    dummy = C.c_void_p(256)                    # never dereferenced: every call below fails its checks first

    def readout(K, B=4, xl=dummy, weights=dummy, D=768):
        return lib_.mtts_adm_readout_mix_f32(xl, D, dummy, K, B, weights, dummy, 1, None, 0, None)
    assert readout(9) == -2 and "K = 9" in lib_.mtts_last_error().decode()
    assert readout(0) == -1
    assert readout(2, weights=None) == -1 and "weights" in lib_.mtts_last_error().decode()
    assert readout(2, xl=None) == -1
    assert readout(2, D=0) == -1
    assert readout(2, B=0) == 0                                           # nothing to do
    assert lib_.mtts_adm_infer_mix_f32(None, 2, None, 0, 0, 1, 1, None, None, None, None, None, 0, None) == -1
    # an ADM descriptor whose pointers are never followed: the K / weights checks come first
    layer = L.EncoderLayer()
    adm = L.ADM()
    adm.enc.layers = C.pointer(layer)
    adm.enc.d_model, adm.emb_dim, adm.tc_emb_dim, adm.tc_dim = 16, 8, 8, 8
    adm.w_dt = adm.w_tc = adm.w_predict = adm.pe = 256

    def mix(K, weights=dummy):
        return lib_.mtts_adm_infer_mix_f32(C.byref(adm), K, dummy, 0, 8, 1, 1, weights, dummy, None, None, dummy, 1 << 30,
                                           None)
    assert mix(9) == -2 and "K = 9" in lib_.mtts_last_error().decode()
    assert mix(0) == -1
    assert mix(2, weights=None) == -1 and "weights" in lib_.mtts_last_error().decode()
    assert lib_.mtts_adm_infer_mix_workspace_bytes(C.byref(adm), 2, 4, 8) > lib_.mtts_adm_infer_workspace_bytes(
        C.byref(adm), 4, 8)
    assert lib_.mtts_adm_infer_mix_workspace_bytes(C.byref(adm), 1, 4, 8) == lib_.mtts_adm_infer_workspace_bytes(
        C.byref(adm), 4, 8)


@pytest.mark.parametrize("raw", [False, True])
def test_infer_mix_calls(lib, raw):  # noqa: F811
    """MegaADM.infer_mix: one workspace query and one mixed decode over the stacked (K*B, T, tc_dim) latents."""
    out = _adm().infer_mix([_latent(), _latent(), _latent()], [1.0, 0.0, 3.0], return_raw=raw)
    assert lib.calls == [
        ("mtts_adm_infer_mix_workspace_bytes", (M_ADM, 3, 2, 5)),
        ("mtts_adm_infer_mix_f32", (M_ADM, 3, P, 40, 8, 2, 5, P, P, P if raw else None, P if raw else None, P, WS_OK,
                                    "stream"))]
    dur = out[0] if raw else out
    assert dur.shape == (2, 5, 1) and dur.dtype == torch.int32
    if raw:
        assert out[1].shape == (2, 5) and out[2].shape == (3, 2, 5) and out[2].dtype == torch.float32


def test_ctypes_signatures_match_the_header():
    """Argument counts of the new entry points in _lib.SIGNATURES against their prototypes in the C header."""
    import os
    from megatts2_b200 import _lib as L
    src = open(os.path.join(ROOT, "include", "megatts2_b200.h")).read()
    for name in ("mtts_adm_readout_mix_f32", "mtts_adm_infer_mix_workspace_bytes", "mtts_adm_infer_mix_f32"):
        m = re.search(r"\b" + name + r"\(([^)]*)\)", src)
        assert m, name
        n_args = len([a for a in m.group(1).split(",") if a.strip()])
        assert len(L.SIGNATURES[name][1]) == n_args, name
        assert L.SIGNATURES[name][0] is (C.c_int64 if name.endswith("_bytes") else C.c_int), name
