"""CPU: duration control's host side - the fitting rule's properties on its exact oracle (tests/ref_duration_control.py),
the validators and the rejected combinations, the entry points MegaADM.infer / infer_mix call with pins, the C argument
checks of the fit (no CUDA call is made) and the ctypes mirror of the new entries."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import ref_duration_control as DC
from conftest import ROOT
from megatts2_b200 import _lib as L
from megatts2_b200 import sampling as S
from test_plm_dispatch_host import M_ADM, P, WS_OK, _adm, _latent, lib  # noqa: F401  (lib: the recorder fixture)


def rng(seed):
    return np.random.default_rng(seed)


def raw_values(r, B, Tp):
    """ADM-like raw values: mostly 1..20 frames, with exact halves, zeros, negatives and ties mixed in."""
    x = (r.gamma(2.0, 3.0, (B, Tp)) + 0.2).astype(np.float32)
    x[:, ::7] = np.float32(2.5)
    x[:, 3::11] = np.float32(-1.0)
    x[:, 5::13] = np.float32(0.0)
    x[:, 1::17] = x[:, :1]
    return x


# ------------------------------------------------------------------------------ the rule
@pytest.mark.parametrize("seed", range(6))
def test_windowed_oracle_equals_the_brute_force_sort(seed):
    r = rng(seed)
    B, Tp = 3, int(r.integers(1, 9))
    raw = raw_values(r, B, Tp)
    if seed % 2:
        raw[1] = np.float32(3.0)                                  # every candidate tied level by level
    pins = np.where(r.random((B, Tp)) < 0.3, r.integers(1, 128, (B, Tp)), -1)
    free = (pins < 1).sum(1)
    psum = np.where(pins >= 1, pins, 0).sum(1)
    for frac in (0.0, 0.13, 0.5, 0.97, 1.0):
        total = (free + psum + np.floor(frac * 127 * free)).astype(np.int64)
        want = DC.fit_brute(raw, 1.0, total, pins)
        assert torch.equal(DC.fit(raw, 1.0, total, pins), want), frac
        assert (want.numpy().sum(1) == total).all()


def test_sum_pins_and_bounds():
    r = rng(10)
    B, Tp = 8, 40
    raw = raw_values(r, B, Tp)
    pins = np.where(r.random((B, Tp)) < 0.25, r.integers(1, 128, (B, Tp)), -1)
    free = (pins < 1).sum(1)
    psum = np.where(pins >= 1, pins, 0).sum(1)
    for total in (free + psum, free + psum + 17, 128 * free + psum, free + psum + 60 * free):
        d = DC.fit(raw, r.uniform(0.5, 2.0, (B, Tp)), total, pins).numpy()
        assert (d.sum(1) == total).all()
        assert (d[pins >= 1] == pins[pins >= 1]).all()
        assert d.min() >= 1 and d.max() <= 128


def test_scale_one_without_a_total_is_the_adm_rounding():
    raw = np.array([[2.5, 1.5, 0.49999997, 0.5, 127.5, 128.49, 1e30, np.inf, -np.inf, np.nan, -0.0, 3.4999998]],
                   np.float32)
    want = [[3, 2, 1, 1, 128, 128, 128, 1, 1, 1, 1, 3]]
    got = DC.fit(raw)
    assert got.tolist() == want
    # the same as (raw + 0.5) -> int32 -> clamp(1, 128) wherever raw is finite (the ADM's own durations; 1e30 is left
    # out, as the CPU's int32 conversion of it is undefined where the device's saturates)
    fin = np.isfinite(raw) & (np.abs(raw) < 1e9)
    adm = (torch.from_numpy(raw) + 0.5).to(torch.int32).clamp(1, 128)
    assert torch.equal(got[torch.from_numpy(fin)], adm[torch.from_numpy(fin)])


@pytest.mark.parametrize("seed", range(4))
def test_theta_one_returns_the_rounding_when_it_already_sums_to_the_total(seed):
    r = rng(20 + seed)
    B, Tp = 6, 64
    raw = raw_values(r, B, Tp)
    scale = r.uniform(0.5, 1.5, (B,)).astype(np.float32)
    pins = np.where(r.random((B, Tp)) < 0.2, r.integers(1, 128, (B, Tp)), -1)
    base = DC.fit(raw, scale, None, pins)
    assert torch.equal(DC.fit(raw, scale, base.sum(1).numpy(), pins), base)


def test_monotone_in_the_total():
    r = rng(30)
    raw = raw_values(r, 2, 30)
    pins = np.full((2, 30), -1)
    pins[1, 4] = 9
    prev = None
    for extra in range(0, 127 * 29 + 1, 97):
        total = np.array([30 + extra, 29 + 9 + min(extra, 127 * 29)])
        d = DC.fit(raw, None, total, pins).numpy()
        if prev is not None:
            assert (d >= prev).all(), extra
        prev = d


def test_ties_go_to_the_lower_phone_index():
    raw = np.full((1, 5), 4.0, np.float32)
    assert DC.fit(raw, None, [6]).tolist() == [[2, 1, 1, 1, 1]]
    assert DC.fit(raw, None, [8]).tolist() == [[2, 2, 2, 1, 1]]
    zeros = np.array([[0.0, -3.0, np.nan, 0.0]], np.float32)              # w = 0 everywhere: phone 0 fills first
    assert DC.fit(zeros, None, [4 + 130]).tolist() == [[128, 4, 1, 1]]
    # equal values across phones: 3/(1 + 1/2) = 2 = 5/(2 + 1/2)
    raw = np.array([[5.0, 3.0]], np.float32)
    assert DC.fit(raw, None, [2 + 2]).tolist() == [[3, 1]]
    assert DC.fit(raw, None, [2 + 3]).tolist() == [[3, 2]]


def test_proportional_to_the_scaled_values():
    """Doubling every scale doubles the durations where nothing saturates (Sainte-Lague is scale-free)."""
    raw = np.array([[3.0, 6.0, 9.0, 12.0]], np.float32)
    assert DC.fit(raw, None, [60]).tolist() == [[6, 12, 18, 24]]
    assert DC.fit(raw, 2.0).tolist() == [[6, 12, 18, 24]]
    assert DC.fit(raw, [[1.0, 1.0, 1.0, 2.0]], [30 + 12]).tolist() == [[3, 6, 9, 24]]


# ------------------------------------------------------------------------------ validators
def test_validators_accept_well_formed_arguments():
    sc, tot, pins = S.duration_control(torch.tensor([1.0, 0.5]), [10, 7], [[-1, 3, -1], [2, -1, -1]], 2, 3)
    assert sc.dtype == torch.float32 and sc.shape == (2,)
    assert tot.dtype == torch.int32 and tot.tolist() == [10, 7]
    assert pins.dtype == torch.int32 and pins.shape == (2, 3)
    assert S.duration_scale(1.25, 2, 3).shape == ()
    assert S.duration_scale(np.ones((2, 3)), 2, 3).shape == (2, 3)
    assert S.duration_control(None, None, None, 2, 3) == (None, None, None)
    # the feasible range edges, [|F| + sum p, 128 |F| + sum p]
    S.total_frames([2 + 3, 128 * 2 + 2], 2, 3, pins)


@pytest.mark.parametrize("kw, match", [
    (dict(scale=0.0), "finite and > 0"), (dict(scale=-1.0), "finite and > 0"), (dict(scale=float("nan")), "finite"),
    (dict(scale=float("inf")), "finite"), (dict(scale=1e-50), "fp32"), (dict(scale=1e39), "fp32"),
    (dict(scale=True), "real number"), (dict(scale=torch.ones(3)), "shape"), (dict(scale="ab"), "duration_scale"),
    (dict(scale=torch.ones(2, 3, 1)), "shape"),
    (dict(pinned=[[0, 1, 1], [1, 1, 1]]), r"pinned_durations\[0, 0\] = 0"),
    (dict(pinned=[[1, 1, 1], [1, 128, 1]]), r"\[1, 1\] = 128"), (dict(pinned=[[-2, 1, 1], [1, 1, 1]]), "-1 .free."),
    (dict(pinned=torch.ones(2, 4, dtype=torch.int32)), "shape"), (dict(pinned=torch.ones(2, 3)), "integers"),
    (dict(total=[2, 3]), r"total_frames\[0\] = 2 is outside utterance 0's feasible range \[3, 384\]"),
    (dict(total=[3, 385]), r"utterance 1's feasible range \[3, 384\]"), (dict(total=[3.0, 3.0]), "integers"),
    (dict(total=[3]), "shape"), (dict(total=[3, 3], pinned=[[5, 5, 5], [-1, -1, -1]]), r"\[15, 15\]"),
    (dict(total=[16, 3], pinned=[[5, 5, 5], [-1, -1, -1]]), "utterance 0"),
])
def test_validators_reject(kw, match):
    args = dict(scale=None, total=None, pinned=None)
    args.update(kw)
    with pytest.raises(L.MttsError, match=match):
        S.duration_control(args["scale"], args["total"], args["pinned"], 2, 3)


def test_fit_bound_on_phones():
    with pytest.raises(L.MttsError, match="8192"):
        S.duration_control(1.5, None, None, 1, 8193)
    S.duration_control(None, None, np.full((1, 8193), -1), 1, 8193)     # pins alone never reach the fit


def test_synthesize_rejects_before_any_device_work():
    """Every rejection happens on the host, with CPU tensors standing in: no device is touched before it."""
    from megatts2_b200.models.megatts2 import Megatts
    tts = Megatts.__new__(Megatts)
    phone = torch.zeros(2, 3, dtype=torch.int64)
    forced = torch.ones(2, 3, dtype=torch.int32)
    for kw in (dict(duration_scale=1.2), dict(total_frames=[3, 3]), dict(pinned_durations=-torch.ones(2, 3))):
        with pytest.raises(L.MttsError, match="forced_durations"):
            tts.synthesize(phone, None, forced_durations=forced, **kw)
        with pytest.raises(L.MttsError, match="forced_durations"):
            tts.synthesize_stream(phone, None, forced_durations=forced, **kw)
    with pytest.raises(L.MttsError, match="causal_decode"):
        tts.synthesize(phone, None, causal_decode=True, pinned_durations=[[1, 2, 3], [-1, -1, 4]])
    for kw in (dict(duration_scale=0.0), dict(total_frames=[2, 3]), dict(pinned_durations=[[0, 1, 1], [1, 1, 1]]),
               dict(duration_scale=torch.ones(2, 4)), dict(total_frames=[[3, 3]])):
        with pytest.raises(L.MttsError):
            tts.synthesize(phone, None, **kw)
        with pytest.raises(L.MttsError):
            tts.synthesize_stream(phone, None, **kw)


def test_synthesize_many_takes_a_scalar_scale_only():
    from megatts2_b200.models.megatts2 import Megatts
    tts = Megatts.__new__(Megatts)
    items = [(torch.zeros(3, dtype=torch.int64), torch.zeros(4, 80))]
    for kw, match in ((dict(duration_scale=torch.ones(1)), "scalar"), (dict(duration_scale=[1.0]), "scalar"),
                      (dict(duration_scale=0.0), "> 0"), (dict(total_frames=[5]), "total_frames"),
                      (dict(pinned_durations=[[1, 1, 1]]), "pinned_durations")):
        with pytest.raises(L.MttsError, match=match):
            tts.synthesize_many(items, **kw)


# ------------------------------------------------------------------------------ dispatch
@pytest.mark.parametrize("raw", [False, True])
def test_infer_with_pins_calls_the_pinned_entry(lib, raw):  # noqa: F811
    out = _adm().infer(_latent(), return_raw=raw, pinned=[[-1, 3, -1, -1, 1], [2, -1, -1, -1, -1]])
    assert lib.calls == [
        ("mtts_adm_infer_mix_workspace_bytes", (M_ADM, 1, 2, 5)),
        ("mtts_adm_infer_pinned_f32", (M_ADM, 1, P, 48, 8, 2, 5, None, 0, 0, P, P if raw else None, None, P, 5, P, WS_OK,
                                       "stream"))]
    dur = out[0] if raw else out
    assert dur.shape == (2, 5, 1) and dur.dtype == torch.int32


@pytest.mark.parametrize("sched", [False, True])
def test_infer_mix_with_pins_calls_the_pinned_entry(lib, sched):  # noqa: F811
    w = torch.ones(2, 5, 3) if sched else [1.0, 0.0, 3.0]
    out = _adm().infer_mix([_latent(), _latent(), _latent()], w, return_raw=True,
                          pinned=torch.full((2, 5), -1, dtype=torch.int32))
    assert lib.calls == [
        ("mtts_adm_infer_mix_workspace_bytes", (M_ADM, 3, 2, 5)),
        ("mtts_adm_infer_pinned_f32", (M_ADM, 3, P, 40, 8, 2, 5, P, *((15, 3) if sched else (3, 0)), P, P, P, P, 5, P,
                                       WS_OK, "stream"))]
    assert out[0].shape == (2, 5, 1) and out[2].shape == (3, 2, 5)


def test_infer_rejects_bad_pins_before_any_call(lib):  # noqa: F811
    for bad in ([[0] * 5, [1] * 5], [[128] * 5, [1] * 5], torch.ones(2, 4, dtype=torch.int64), torch.ones(2, 5)):
        with pytest.raises(L.MttsError, match="pinned_durations"):
            _adm().infer(_latent(), pinned=bad)
        with pytest.raises(L.MttsError, match="pinned_durations"):
            _adm().infer_mix([_latent(), _latent()], [1.0, 1.0], pinned=bad)
    assert lib.calls == []


# ------------------------------------------------------------------------------ C side
def test_c_side_rejects_bad_fit_arguments():
    """mtts_fit_durations_f32 validates before it enqueues anything (so no device is needed to see the errors)."""
    lib_ = L.lib()
    dummy = C.c_void_p(256)                    # never dereferenced: every call below fails its checks first

    def fit(Tp=4, B=2, raw=dummy, out=dummy, raw_sb=4, sc_sb=0, sc_st=0, pin_sb=4, dur_sb=4):
        return lib_.mtts_fit_durations_f32(raw, raw_sb, Tp, B, None, sc_sb, sc_st, None, pin_sb, None, out, dur_sb, None)
    assert fit(Tp=0) == -1
    assert fit(Tp=8193) == -2 and "8192" in lib_.mtts_last_error().decode()
    assert fit(raw_sb=-1) == -1 and fit(sc_st=-1) == -1 and fit(pin_sb=-1) == -1 and fit(dur_sb=-1) == -1
    assert fit(raw=None) == -1 and fit(out=None) == -1
    assert fit(B=0) == 0                                                  # nothing to do
    assert lib_.mtts_adm_infer_pinned_f32(None, 1, None, 0, 0, 1, 1, None, 0, 0, None, None, None, None, 0, None, 0,
                                          None) == -1


def test_ctypes_signatures_match_the_header():
    """Argument counts of the new entry points in _lib.SIGNATURES against their prototypes in the C header."""
    import os
    src = open(os.path.join(ROOT, "include", "megatts2_b200.h")).read()
    for name in ("mtts_adm_infer_pinned_f32", "mtts_fit_durations_f32"):
        m = re.search(r"\b" + name + r"\(([^)]*)\)", src)
        assert m, name
        n_args = len([a for a in m.group(1).split(",") if a.strip()])
        assert len(L.SIGNATURES[name][1]) == n_args, name
        assert L.SIGNATURES[name][0] is C.c_int, name
