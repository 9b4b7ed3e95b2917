"""CPU: timbre interpolation's host side - every validation error of Megatts.synthesize / synthesize_stream's timbre
arguments and of MRTE.tc_latent_mix, the rejections by edit and synthesize_many, the entries the synthesis MRTE pass and
tc_latent_mix call (the library replaced by a recorder), the fp64 restatement's rules, the C argument checks and the
ctypes mirror of mtts_mix_layernorm_f32."""
import ctypes as C
import functools
import os
import re

import numpy as np
import pytest
import torch

import ref_timbre_mix as RT
from conftest import ROOT
from megatts2_b200 import _lib as L
from megatts2_b200 import graphs, ops
from megatts2_b200.edit import REJECTED
from megatts2_b200.models.megatts2 import Megatts
from megatts2_b200.modules.mrte import MRTE

B, TP, NB = 2, 5, 80


class Recorder:
    """Stands in for the library: records the entry names (and the integer arguments of mtts_mix_layernorm_f32), returns
    4096 for a workspace query, the strided conv's length for mtts_convnet_double_out_len, else 0."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return functools.partial(self._call, name)

    def _call(self, name, *args):
        assert len(args) == len(L.SIGNATURES[name][1]), name
        if name == "mtts_mix_layernorm_f32":
            self.calls.append((name, tuple(a for a, t in zip(args, L.SIGNATURES[name][1]) if t in (C.c_int32, C.c_int64))))
        else:
            self.calls.append(name)
        if name.endswith("_workspace_bytes") or name == "mtts_linear_tc_scratch_bytes":
            return 4096
        if name == "mtts_convnet_double_out_len":
            return (args[1] - 1) // 16 + 1
        return 0


@pytest.fixture
def lib(monkeypatch):
    rec = Recorder()
    monkeypatch.setattr(L, "lib", lambda: rec)
    monkeypatch.setattr(ops, "_dev", lambda t, dtype=torch.float32, name="tensor": _cpu_dev(t, dtype, name))
    monkeypatch.setattr(ops, "workspace", lambda nbytes, device: torch.empty(int(nbytes) + 256, dtype=torch.uint8))
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0x5EA))
    monkeypatch.setattr(ops, "tc_overflow_bind", lambda device: None)
    monkeypatch.setattr(graphs, "_enabled", False)
    return rec


def _cpu_dev(t, dtype, name):
    if not isinstance(t, torch.Tensor) or t.dtype != dtype:
        raise L.MttsError(f"{name}: expected a {dtype} tensor")
    return t


def _mrte():
    return MRTE(hidden_size=32, content_ff_dim=64, content_n_layers=1, mel_n_layer=1, mel_n_stack=1,
                mel_n_block=1).eval()


def _tts(mrte=None):
    tts = Megatts.__new__(Megatts)
    torch.nn.Module.__init__(tts)
    tts.generator = type("G", (), {"mrte": mrte if mrte is not None else _mrte()})()
    return tts


def _phone():
    return torch.randint(0, 320, (B, TP))


def _mel(T=40):
    return torch.randn(B, T, NB)


# ------------------------------------------------------------------------------ validation
@pytest.mark.parametrize("kw, match", [
    (dict(timbre_weights=[1.0, 1.0]), "timbre_weights without timbre_mels"),
    (dict(timbre_mels=["m"]), "timbre_mels needs timbre_weights"),
    (dict(timbre_mels=[], timbre_weights=[1.0]), "timbre_mels must be a non-empty list"),
    (dict(timbre_mels="tensor", timbre_weights=[1.0, 1.0]), "timbre_mels must be a non-empty list"),
    (dict(timbre_mels=["m"] * 8, timbre_weights=[1.0] * 9), r"timbre_mels: 8 prompts, at most 7"),
    (dict(timbre_mels=["m"], timbre_weights=[1.0]), r"timbre_weights: weights of shape \(1,\)"),
    (dict(timbre_mels=["m"], timbre_weights=[1.0, 1.0, 1.0]), r"timbre_weights: weights of shape \(3,\)"),
    (dict(timbre_mels=["m"], timbre_weights=[[1.0, 1.0]] * 3), r"timbre_weights: weights of shape \(3, 2\)"),
    (dict(timbre_mels=["m"], timbre_weights=[1.0, -0.5]), r"timbre_weights: weight \[0, 1\] = -0.5"),
    (dict(timbre_mels=["m"], timbre_weights=[[1.0, 0.0], [float("nan"), 1.0]]), r"timbre_weights: weight \[1, 0\] = nan"),
    (dict(timbre_mels=["m"], timbre_weights=[float("inf"), 1.0]), r"timbre_weights: weight \[0, 0\] = inf"),
    (dict(timbre_mels=["m"], timbre_weights=[[1.0, 0.0], [0.0, 0.0]]), r"timbre_weights: weight row \[1\] sums to 0"),
    (dict(timbre_mels=["m"], timbre_weights=[3e38, 3e38]), r"timbre_weights: weight row \[0\] sums to inf"),
    (dict(timbre_mels=["m"], timbre_weights="sched_bad_row"), r"timbre_weights: weight row \[1, 3\] sums to 0"),
    (dict(timbre_mels=["m"], timbre_weights=np.ones((B, TP + 1, 2))), r"timbre_weights: weights of shape \(2, 6, 2\), "
                                                                       r"expected \(2, 5, 2\)"),
    (dict(timbre_mels=["m"], timbre_weights=np.ones((B, TP, 3))), r"timbre_weights: weights of shape \(2, 5, 3\)"),
    (dict(timbre_mels=["short"], timbre_weights=[1.0, 1.0]), r"timbre_mels\[0\]: expected \(2, Tm, 80\), got \(1, 40, 80\)"),
    (dict(timbre_mels=["m", "bins"], timbre_weights=[1.0, 1.0, 1.0]), r"timbre_mels\[1\]: expected \(2, Tm, 80\)"),
    (dict(timbre_mels=["empty"], timbre_weights=[1.0, 1.0]), r"timbre_mels\[0\]: expected \(2, Tm, 80\), got \(2, 0, 80\)"),
    (dict(timbre_mels=["f64"], timbre_weights=[1.0, 1.0]), r"timbre_mels\[0\]: expected a torch.float32"),
])
@pytest.mark.parametrize("entry", ["synthesize", "synthesize_stream"])
def test_synthesize_rejects_bad_timbre_arguments(lib, kw, match, entry):
    prompts = {"m": _mel(), "short": torch.zeros(1, 40, NB), "bins": torch.zeros(B, 40, 81),
               "empty": torch.zeros(B, 0, NB), "f64": torch.zeros(B, 40, NB, dtype=torch.float64)}
    kw = dict(kw)
    if isinstance(kw.get("timbre_mels"), list):
        kw["timbre_mels"] = [prompts[m] for m in kw["timbre_mels"]]
    elif kw.get("timbre_mels") == "tensor":
        kw["timbre_mels"] = _mel()
    if isinstance(kw.get("timbre_weights"), str):
        w = torch.ones(B, TP, 2)
        w[1, 3] = 0.0
        kw["timbre_weights"] = w
    tts = _tts()
    with pytest.raises(L.MttsError, match=match):
        getattr(tts, entry)(_phone(), _mel(), **kw)
    assert lib.calls == []                      # checked on the host before any device work


def test_valid_timbre_arguments_reach_the_synthesis_body(lib, monkeypatch):
    seen = []
    monkeypatch.setattr(Megatts, "_synthesize", lambda self, *a, timbre=None: seen.append(timbre) or {"wav": None})
    tts, p = _tts(), _mel(33)
    tts.synthesize(_phone(), _mel(), check_range=False)
    tts.synthesize(_phone(), _mel(), check_range=False, timbre_mels=[p], timbre_weights=[0.25, 0.75])
    tts.synthesize(_phone(), _mel(), check_range=False, timbre_mels=(p, p), timbre_weights=torch.rand(B, TP, 3) + 0.1)
    assert seen[0] is None
    assert seen[1][0][0] is p and seen[1][1].tolist() == [[0.25, 0.75]] * B
    assert seen[2][1].shape == (B, TP, 3) and len(seen[2][0]) == 2
    assert lib.calls == []


@pytest.mark.parametrize("name", ["timbre_mels", "timbre_weights"])
def test_edit_rejects_timbre_by_name(name):
    assert name in REJECTED
    tts = _tts()
    ph = torch.tensor([[1, 2, 3]])
    with pytest.raises(L.MttsError, match=f"edit does not take {name}"):
        tts.edit(ph, None, ph, torch.ones(1, 3, dtype=torch.int64), torch.zeros(1, 1, dtype=torch.int64),
                 torch.tensor([[0, 1]]), **{name: [1.0, 1.0]})


@pytest.mark.parametrize("kw", [dict(timbre_mels=[torch.zeros(1, 4, NB)]), dict(timbre_weights=[1.0, 1.0])])
def test_synthesize_many_rejects_timbre(kw):
    with pytest.raises(L.MttsError, match="synthesize_many does not take timbre_mels or timbre_weights"):
        _tts().synthesize_many([(torch.zeros(3, dtype=torch.int64), torch.zeros(4, NB))], **kw)


@pytest.mark.parametrize("mels, weights, match", [
    ([], [1.0], "non-empty list"),
    ("tensor", [1.0], "non-empty list"),
    (["m"] * 9, [1.0] * 9, "K = 9 sources"),
    (["m", "m"], [1.0], r"weights of shape \(1,\)"),
    (["m", "m"], [1.0, float("nan")], r"weight \[0, 1\] = nan"),
    (["m", "m"], [0.0, 0.0], r"weight row \[0\] sums to 0"),
    (["m", "short"], [1.0, 1.0], r"mels\[1\]: expected \(2, Tm, 80\)"),
])
def test_tc_latent_mix_rejects(lib, mels, weights, match):
    prompts = {"m": _mel(), "short": torch.zeros(1, 40, NB)}
    mels = _mel() if mels == "tensor" else [prompts[m] for m in mels]
    with pytest.raises(L.MttsError, match=match):
        _mrte().tc_latent_mix(_phone(), mels, weights)
    assert lib.calls == []


# ------------------------------------------------------------------------------ dispatch
def _count(calls, name):
    return sum(1 for c in calls if (c if isinstance(c, str) else c[0]) == name)


def test_mrte_pass_without_prompts_is_tc_latent(lib):
    mrte = _mrte()
    ph, mel = _phone(), _mel()
    mrte.tc_latent(ph, mel)
    want = list(lib.calls)
    lib.calls.clear()
    tc, pros, blend = _tts(mrte)._mrte(ph, mel, None, None)
    assert lib.calls == want and pros is None and blend is None and tc.shape == (B, TP, 32)


def _timbre(tts, ph, mels, weights):
    return tts._check_timbre(ph, mels, weights)


def test_tc_latent_mix_runs_the_phone_encoder_once(lib):
    mrte = _mrte()
    ph, mels = _phone(), [_mel(), _mel(17), _mel(64)]
    out = mrte.tc_latent_mix(ph, mels, torch.rand(B, TP, 3) + 0.1)
    assert out.shape == (B, TP, 32)
    assert _count(lib.calls, "mtts_encoder_forward_f32") == 1
    assert _count(lib.calls, "mtts_convnet_double_forward_f32") == 3
    assert _count(lib.calls, "mtts_layernorm_f32") == 0
    mix = [c for c in lib.calls if not isinstance(c, str)]
    # (y_ks, ldy, K, w_sb, w_st, T, ldo, rows, C, post_act): per-phone weights at strides (T K, K)
    assert mix == [("mtts_mix_layernorm_f32", (B * TP * 32, 32, 3, TP * 3, 3, TP, 32, B * TP, 32, L.ACT_RELU))]
    lib.calls.clear()
    mrte.tc_latent_mix(ph, mels[:2], [1.0, 2.0])
    assert [c for c in lib.calls if not isinstance(c, str)][0][1][3:5] == (2, 0)      # (K,) -> the (B, K) rows


@pytest.mark.parametrize("shared", [False, True])
def test_mrte_pass_encodes_each_prompt_once(lib, shared):
    mrte = _mrte()
    tts = _tts(mrte)
    ph, mel, t1, p1 = _phone(), _mel(), _mel(24), _mel(48)
    pros = [t1 if shared else _mel(24), p1]
    timbre = _timbre(tts, ph, [t1], [0.4, 0.6])
    tc, lats, blend = tts._mrte(ph, mel, pros, timbre)
    assert len(lats) == 2 and blend.shape == tc.shape == (B, TP, 32)
    assert _count(lib.calls, "mtts_encoder_forward_f32") == 1
    assert _count(lib.calls, "mtts_convnet_double_forward_f32") == (3 if shared else 4)
    assert _count(lib.calls, "mtts_layernorm_f32") == 3                  # the target's and the two prosody latents
    assert _count(lib.calls, "mtts_mix_layernorm_f32") == 1
    if shared:                                                          # one latent serves the prompt in both roles
        assert lats[0] is not tc


def test_mrte_pass_with_prosody_only_and_repeats(lib):
    mrte = _mrte()
    ph, mel, p = _phone(), _mel(), _mel(24)
    tc, lats, blend = _tts(mrte)._mrte(ph, mel, [p, mel, p], None)
    assert blend is None and lats[0] is lats[2] and lats[1] is tc
    assert _count(lib.calls, "mtts_encoder_forward_f32") == 1
    assert _count(lib.calls, "mtts_convnet_double_forward_f32") == 2
    assert _count(lib.calls, "mtts_layernorm_f32") == 2 and _count(lib.calls, "mtts_mix_layernorm_f32") == 0


# ------------------------------------------------------------------------------ the restatement's rules
def test_restatement_rules():
    g = torch.Generator().manual_seed(3)
    ys = torch.randn(3, 2, 4, 16, generator=g, dtype=torch.float64)
    gamma, beta = torch.randn(16, generator=g), torch.randn(16, generator=g)
    one = RT.mix_layernorm(ys, [0.0, 2.0, 0.0], gamma, beta)
    assert torch.allclose(one, torch.relu(torch.nn.functional.layer_norm(ys[1], (16,), gamma.double(), beta.double())))
    poisoned = ys.clone()
    poisoned[0] = float("nan")
    poisoned[2] = float("inf")
    assert torch.equal(RT.mix_layernorm(poisoned, [0.0, 2.0, 0.0], gamma, beta), one)
    half = RT.mix_layernorm(ys, [1.0, 1.0, 0.0], gamma, beta)
    assert torch.allclose(half, RT.mix_layernorm(ys, [3.0, 3.0, 0.0], gamma, beta))
    sched = torch.tensor([[0.0, 1.0, 0.0]] * 4)[None].repeat(2, 1, 1)
    assert torch.equal(RT.mix_layernorm(ys, sched, gamma, beta), RT.mix_layernorm(ys, [0.0, 1.0, 0.0], gamma, beta))


# ------------------------------------------------------------------------------ C side
def _err():
    return L.lib().mtts_last_error().decode()


def test_c_side_rejects_bad_mix_layernorm_arguments():
    """mtts_mix_layernorm_f32 checks every argument before it enqueues anything (so no device is needed to see the
    errors)."""
    lib_ = L.lib()
    dummy = C.c_void_p(256)                    # never dereferenced: every call below fails its checks first

    def call(y=dummy, y_ks=2048, ldy=512, K=2, w=dummy, w_sb=2, w_st=0, T=4, g=dummy, b=dummy, out=dummy, ldo=512,
             rows=8, Cc=512, act=L.ACT_RELU):
        return lib_.mtts_mix_layernorm_f32(y, y_ks, ldy, K, w, w_sb, w_st, T, g, b, out, ldo, rows, Cc, 1e-5, act, None)
    assert call(K=9) == -2 and "K = 9" in _err()
    assert call(K=0) == -1 and "K" in _err()
    for c in (128, 256, 500, 2048):
        assert call(Cc=c, ldy=c, ldo=c) == -2 and f"C = {c}" in _err()
    assert call(rows=-1) == -1 and "rows" in _err()
    for kw in (dict(y=None), dict(w=None), dict(g=None), dict(b=None), dict(out=None)):
        assert call(**kw) == -1 and "null" in _err(), kw
    for kw in (dict(T=0), dict(y_ks=-4), dict(w_sb=-1), dict(w_st=-1), dict(ldy=508), dict(ldo=100)):
        assert call(**kw) == -1 and "strides" in _err(), kw
    assert call(act=L.ACT_LEAKY) == -1 and "post_act" in _err()
    for kw in (dict(y=C.c_void_p(260)), dict(out=C.c_void_p(264)), dict(ldy=514), dict(y_ks=2050)):
        assert call(**kw) == -1 and "aligned" in _err(), kw
    assert call(rows=0) == 0                                                # nothing to do


def test_ctypes_signature_matches_the_header():
    src = open(os.path.join(ROOT, "include", "megatts2_b200.h")).read()
    name = "mtts_mix_layernorm_f32"
    m = re.search(r"\b" + name + r"\(([^)]*)\)", src)
    assert m
    args = [a.strip() for a in m.group(1).split(",") if a.strip()]
    types = L.SIGNATURES[name][1]
    assert len(types) == len(args) and L.SIGNATURES[name][0] is C.c_int
    want = {"int64_t": C.c_int64, "int32_t": C.c_int32, "float": C.c_float}
    for a, t in zip(args, types):
        base = a.rsplit(" ", 1)[0].replace("const ", "")
        assert t is (C.c_void_p if "*" in a else want[base]), a
    assert getattr(L.lib(), name) is not None
