"""CPU: the host side of mix schedules (per-step and per-phone prosody and duration weights) - the phone -> PLM step rule
of tests/ref_mix_schedule.py on hand-worked cases, the (B, T, K) validator, the entry points MegaPLM / MegaADM call with
schedules and their strides, the argument checks of the new C entries (no CUDA call is made), and their ctypes mirror."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import ref_mix_schedule as MS
from conftest import ROOT
from megatts2_b200 import _lib as L
from megatts2_b200 import sampling as S
from test_plm_dispatch_host import M_ADM, M_PLM, P, SMP_STRUCT, WS_OK, _adm, _latent, _plm, _smp, lib  # noqa: F401


# ------------------------------------------------------------------------------ the step rule
@pytest.mark.parametrize("durations, T, want", [
    ([[8, 8]], 2, [[0, 1]]),                               # one phone per step
    ([[4, 4, 8]], 2, [[0, 2]]),                            # a tie: the earlier phone
    ([[3, 5, 8]], 2, [[1, 2]]),                            # the majority
    ([[2, 3, 3, 8]], 2, [[1, 3]]),                         # a tie between later phones: the earlier of them
    ([[5, 0, 0, 11]], 2, [[0, 3]]),                        # zero-duration phones own no frames
    ([[0, 8, 0]], 3, [[1, 1, 1]]),                         # steps past the end: the last phone with a duration
    ([[4, 6, 0, 0]], 4, [[0, 1, 1, 1]]),                   # a 4-4 tie, a partial last step, then past the end
    ([[0, 0, 0]], 2, [[0, 0]]),                            # L = 0: phone 0
    ([[-3, 8, -1]], 2, [[1, 1]]),                          # negative durations count as 0
    ([[13]], 3, [[0, 0, 0]]),                              # Tp = 1
    ([[8, 8, 8], [20, 0, 1]], 3, [[0, 1, 2], [0, 0, 0]]),  # ragged totals: the shorter utterance repeats its last phone
    ([[1, 1, 1, 1, 1, 1, 1, 1, 2, 6]], 2, [[0, 9]]),       # eight one-frame phones tie: the first
])
def test_step_rule_cases(durations, T, want):
    assert MS.step_phones(durations, T).tolist() == want


def test_step_rule_random_against_frame_counts():
    """Random durations: every step's phone owns at least as many of its frames as any other, and strictly more than
    every earlier one."""
    rng = np.random.default_rng(3)
    for _ in range(200):
        B, Tp = int(rng.integers(1, 4)), int(rng.integers(1, 30))
        d = rng.integers(-1, 12, (B, Tp))
        d[rng.random((B, Tp)) < 0.2] = 0
        T = int(-(-np.maximum(d, 0).sum(1).max() // 8)) + int(rng.integers(0, 3))
        got = MS.step_phones(d, T)
        for b in range(B):
            owner = np.repeat(np.arange(Tp), np.maximum(d[b], 0))
            for t in range(T):
                fr = owner[8 * t:8 * t + 8]
                if not fr.size:
                    assert got[b, t] == (owner[-1] if owner.size else 0)
                    continue
                cnt = np.bincount(fr, minlength=Tp)
                p = got[b, t]
                assert cnt[p] == cnt.max() and (cnt[:p] < cnt[p]).all()
    pw = rng.random((2, 5, 3)).astype(np.float32)
    d = np.array([[8, 0, 16, 1, 7], [3, 3, 3, 3, 3]])
    assert np.array_equal(MS.step_weights(pw, d, 4), pw[np.arange(2)[:, None], MS.step_phones(d, 4)])


# ------------------------------------------------------------------------------ validator
def test_step_weight_validator():
    w = S.mix_step_weights(torch.tensor([[[1.0, 0.0], [0.25, 0.75], [0.0, 3.0]]]), 2, 1, 3)
    assert w.dtype == torch.float32 and w.shape == (1, 3, 2) and w.is_contiguous() and w.device.type == "cpu"
    assert S.mix_step_weights(np.ones((2, 4, 3), np.int32), 3, 2, 4).dtype == torch.float32
    assert S.mix_step_weights(np.ones((0, 4, 3)), 3, 0, 4).shape == (0, 4, 3)
    bad = [np.ones((1, 3, 2)),                    # wrong B
           np.ones((2, 4, 2)),                    # wrong T
           np.ones((2, 3, 3)),                    # wrong K
           np.ones((2, 3)),                       # per utterance, not a schedule
           [[[1.0, -1.0]] * 3] * 2,               # negative
           [[[1.0, float("nan")]] * 3] * 2,       # NaN
           [[[1.0, float("inf")]] * 3] * 2,       # inf
           [[[1.0, 1.0], [0.0, 0.0], [1.0, 1.0]]] * 2,   # a row without a positive weight
           np.full((2, 3, 2), 3e38, np.float64),  # the fp32 row sum overflows
           np.ones((2, 3, 2), bool), "abc"]
    for w in bad:
        with pytest.raises(L.MttsError, match="prosody mix"):
            S.mix_step_weights(w, 2, 2, 3)
    with pytest.raises(L.MttsError, match="K = 9"):
        S.mix_step_weights(np.ones((1, 2, 9)), 9, 1, 2)
    assert S.per_step(np.ones((1, 2, 3))) and not S.per_step([1.0, 2.0]) and not S.per_step(np.ones((2, 3)))
    assert not S.per_step("abc") and not S.per_step(None)


def test_synthesize_routes_weights_by_rank(monkeypatch):
    """_check_prosody takes (B, Tp, K) prosody and duration weights and keeps every per-utterance rejection."""
    from megatts2_b200 import ops
    from megatts2_b200.models.megatts2 import Megatts
    monkeypatch.setattr(ops, "_dev", lambda t, dtype=torch.float32, name="tensor": t)
    tts = Megatts.__new__(Megatts)
    tts.generator = type("G", (), {"mrte": type("M", (), {"mel_bins": 80})()})()
    phone = torch.zeros(2, 3, dtype=torch.int64)
    pros = [torch.zeros(2, 4, 80)]
    sched = torch.rand(2, 3, 2) + 0.1
    tts._check_prosody(phone, pros, sched, False, sched)
    tts._check_prosody(phone, pros, [1.0, 1.0], False, sched)
    tts._check_prosody(phone, pros, sched, False, [0.5, 0.5])
    for bad in (torch.ones(2, 4, 2), torch.ones(3, 3, 2), torch.ones(2, 3, 3), -sched):
        with pytest.raises(L.MttsError, match="prosody mix"):
            tts._check_prosody(phone, pros, bad, False)
        with pytest.raises(L.MttsError, match="duration mix"):
            tts._check_prosody(phone, pros, [1.0, 1.0], False, bad)
    with pytest.raises(L.MttsError, match="causal"):
        tts._check_prosody(phone, pros, sched, True)


# ------------------------------------------------------------------------------ dispatch
def _sched(T=5, K=2):
    return torch.rand(2, T, K) + 0.1


@pytest.mark.parametrize("rl", [False, True])
@pytest.mark.parametrize("sampled", [False, True])
def test_infer_mix_schedule_calls(lib, sampled, rl):  # noqa: F811
    out = _plm().infer_mix([_latent(), _latent()], _sched(), return_logits=rl, **_smp(sampled))
    assert lib.calls == [
        ("mtts_plm_infer_mix_workspace_bytes", (M_PLM, 2, 2, 5)),
        ("mtts_plm_infer_mix_steps_f32", (M_PLM, 2, P, 40, 8, 2, 5, P, 10, 2, P, P if rl else None,
                                          SMP_STRUCT if sampled else None, P, WS_OK, "stream"))]
    if rl:
        assert out[1].shape == (2, 2, 5, 16)


@pytest.mark.parametrize("sampled", [False, True])
def test_decode_until_schedule_calls(lib, sampled):  # noqa: F811
    plm = _plm()
    dec = plm.begin_decode([_latent(), _latent(), _latent()], weights=_sched(K=3), **_smp(sampled))
    assert dec.K == 3 and lib.calls == []
    plm.decode_until(dec, 2)
    plm.decode_until(dec, 2)
    c, lg = plm.decode_until(dec, 5, return_logits=True)
    assert lg.shape == (3, 2, 3, 16) and plm.decode_until(dec, 5, return_logits=True)[1].shape == (3, 2, 0, 16)

    def steps(t0, t1, rl):
        return [("mtts_plm_infer_mix_workspace_bytes", (M_PLM, 3, 2, 5)),
                ("mtts_plm_infer_mix_steps_range_f32", (M_PLM, 3, P, 40, 8, 2, 5, P, 15, 3, t0, t1, P, P,
                                                        P if rl else None, SMP_STRUCT if sampled else None, P, WS_OK,
                                                        "stream"))]
    assert lib.calls == steps(0, 2, False) + steps(2, 5, True)


@pytest.mark.parametrize("raw", [False, True])
def test_adm_infer_mix_schedule_calls(lib, raw):  # noqa: F811
    out = _adm().infer_mix([_latent(), _latent(), _latent()], _sched(K=3), return_raw=raw)
    assert lib.calls == [
        ("mtts_adm_infer_mix_workspace_bytes", (M_ADM, 3, 2, 5)),
        ("mtts_adm_infer_mix_steps_f32", (M_ADM, 3, P, 40, 8, 2, 5, P, 15, 3, P, P if raw else None, P if raw else None,
                                          P, WS_OK, "stream"))]
    assert (out[0] if raw else out).shape == (2, 5, 1)


def test_per_utterance_weights_keep_the_old_entries(lib):  # noqa: F811
    plm, adm = _plm(), _adm()
    for w in ([1.0, 3.0], torch.tensor([[1.0, 3.0], [2.0, 0.0]])):
        plm.infer_mix([_latent(), _latent()], w)
        adm.infer_mix([_latent(), _latent()], w)
        dec = plm.begin_decode([_latent(), _latent()], weights=w)
        plm.decode_until(dec, 5)
    names = [c[0] for c in lib.calls if not c[0].endswith("_bytes")]
    assert names == ["mtts_plm_infer_mix_f32", "mtts_adm_infer_mix_f32", "mtts_plm_infer_mix_range_f32"] * 2


def test_schedule_and_row_mixes_are_separate_graphs(lib, monkeypatch):  # noqa: F811
    from megatts2_b200 import graphs
    monkeypatch.setattr(graphs, "_enabled", True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    plm, adm = _plm(), _adm()
    plm.infer_mix([_latent(), _latent()], [1.0, 3.0])
    plm.infer_mix([_latent(), _latent()], _sched())
    adm.infer_mix([_latent(), _latent()], [1.0, 3.0])
    adm.infer_mix([_latent(), _latent()], _sched())
    assert len(plm._graphs().cache) == 2 and len(adm._graphs().cache) == 2


def test_schedule_shape_is_checked(lib):  # noqa: F811
    for w in (torch.ones(2, 4, 2), torch.ones(2, 5, 3), torch.ones(1, 5, 2)):
        with pytest.raises(L.MttsError, match="prosody mix"):
            _plm().infer_mix([_latent(), _latent()], w)
        with pytest.raises(L.MttsError, match="duration mix"):
            _adm().infer_mix([_latent(), _latent()], w)
    assert lib.calls == []


# ------------------------------------------------------------------------------ C argument checks
def _err():
    return L.lib().mtts_last_error().decode()


def test_c_entries_reject_bad_arguments():
    """The new entries validate before they enqueue anything, so no device is needed to see the errors."""
    lib_ = L.lib()
    dummy = C.c_void_p(256)                    # never dereferenced: every call below fails its checks first

    def expand(K=2, Tp=4, B=1, T=2, pw=dummy, pw_sb=8, dur=dummy, dur_sb=4, out=dummy):
        return lib_.mtts_mix_step_weights_f32(pw, pw_sb, Tp, K, B, dur, dur_sb, T, out, None)
    assert expand(K=9) == -2 and "K = 9" in _err()
    assert expand(K=0) == -1
    assert expand(Tp=0) == -1 and "Tp" in _err()
    assert expand(Tp=8193) == -2 and "Tp = 8193" in _err()
    assert expand(pw_sb=-1) == -1 and "strides" in _err()
    assert expand(dur_sb=-4) == -1 and "strides" in _err()
    for kw in (dict(pw=None), dict(dur=None), dict(out=None)):
        assert expand(**kw) == -1 and "null" in _err()
    assert expand(T=0) == 0 and expand(B=0) == 0 and expand(T=-1, out=None) == 0     # nothing to do

    layer = L.EncoderLayer()
    plm = L.PLM()
    plm.enc.layers = C.pointer(layer)
    plm.enc.d_model, plm.vq_dim, plm.tc_dim, plm.vq_bins = 16, 8, 8, 16
    plm.pc_embedding = plm.w_predict = plm.pe = 256
    adm = L.ADM()
    adm.enc.layers = C.pointer(layer)
    adm.enc.d_model, adm.emb_dim, adm.tc_emb_dim, adm.tc_dim = 16, 8, 8, 8
    adm.w_dt = adm.w_tc = adm.w_predict = adm.pe = 256

    def plm_whole(K=2, w=dummy, w_sb=10, w_st=2, ws=dummy):
        return lib_.mtts_plm_infer_mix_steps_f32(C.byref(plm), K, dummy, 0, 8, 1, 5, w, w_sb, w_st, dummy, None, None,
                                                 ws, 1 << 30, None)

    def plm_range(K=2, w=dummy, w_sb=10, w_st=2, t0=0, t1=5, state=dummy):
        return lib_.mtts_plm_infer_mix_steps_range_f32(C.byref(plm), K, dummy, 0, 8, 1, 5, w, w_sb, w_st, t0, t1, state,
                                                       dummy, None, None, dummy, 1 << 30, None)

    def adm_mix(K=2, w=dummy, w_sb=10, w_st=2, ws=dummy):
        return lib_.mtts_adm_infer_mix_steps_f32(C.byref(adm), K, dummy, 0, 8, 1, 5, w, w_sb, w_st, dummy, None, None,
                                                 ws, 1 << 30, None)
    for entry in (plm_whole, plm_range, adm_mix):
        assert entry(K=9) == -2 and "K = 9" in _err(), entry.__name__
        assert entry(K=0) == -1, entry.__name__
        assert entry(w=None) == -1 and "null" in _err(), entry.__name__
        assert entry(w_sb=-1) == -1 and "strides" in _err(), entry.__name__
        assert entry(w_st=-2) == -1 and "strides" in _err(), entry.__name__
    assert plm_whole(ws=None) == -1 and adm_mix(ws=None) == -1
    assert plm_range(t0=3, t1=2) == -1 and "range" in _err()
    assert plm_range(state=None) == -1
    assert lib_.mtts_plm_infer_mix_steps_f32(None, 2, dummy, 0, 8, 1, 5, dummy, 10, 2, dummy, None, None, dummy, 1, None) == -1
    assert lib_.mtts_adm_infer_mix_steps_f32(None, 2, dummy, 0, 8, 1, 5, dummy, 10, 2, dummy, None, None, dummy, 1, None) == -1


def test_ctypes_signatures_match_the_header():
    import os
    src = open(os.path.join(ROOT, "include", "megatts2_b200.h")).read()
    for name in ("mtts_plm_infer_mix_steps_f32", "mtts_plm_infer_mix_steps_range_f32", "mtts_adm_infer_mix_steps_f32",
                 "mtts_mix_step_weights_f32"):
        m = re.search(r"\b" + name + r"\(([^)]*)\)", src)
        assert m, name
        assert len(L.SIGNATURES[name][1]) == len([a for a in m.group(1).split(",") if a.strip()]), name
        assert L.SIGNATURES[name][0] is C.c_int, name
        assert getattr(L.lib(), name) is not None
