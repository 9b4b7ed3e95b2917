"""GPU: duration control.  The fit kernel (csrc/ops.cu, fit_durations_kernel) against its exact oracle
(tests/ref_duration_control.py), pinned ADM decodes against the unpinned ones and the fp64 restatement, and
Megatts.synthesize / synthesize_stream with duration_scale, total_frames and pinned_durations.

Bars: the fit bit for bit; all-free pins, one-hot mixes and graph replays bit for bit; pinned phones exactly their pin;
the free phones' raw values within RAW_REL = 2e-3 of the fp64 oracle, relative to max(1, max |raw|), and their durations
equal except where the fp64 value lies within 1e-4 of a rounding boundary (test_gpu_duration_mix.py's bars)."""
import numpy as np
import pytest
import torch

import helpers
import ref_duration_control as DC
from megatts2_b200 import _lib as L
from megatts2_b200 import graphs, ops, pack
from megatts2_b200.sampling import Sampling
from oracle import weights
from test_gpu_duration_mix import RAW_REL, NEAR, _boundary_distance, sources

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda"
ENGINES = pytest.mark.parametrize("engine", [pack.ENGINE_F16X2, pack.ENGINE_BF16X3, pack.ENGINE_FFMA],
                                  ids=["f16x2", "bf16x3", "ffma"])


def gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def tts(weights_cpu):
    return helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)


# ------------------------------------------------------------------------------ the fit kernel
def fit_case(B, Tp, seed, pinned):
    """Raw values with equal values, exact half-integers, w <= 0, NaN and +-inf; pins on about a quarter of the phones;
    totals with N = 0 (row 0), N = 127 |F| (row 1), the no-total sum (row 2) and random feasible ones."""
    r = np.random.default_rng(seed)
    raw = (r.gamma(2.0, 3.0, (B, Tp)) + 0.1).astype(np.float32)
    raw[:, ::5] = np.float32(4.0)
    raw[:, 2::9] = (r.integers(0, 30, raw[:, 2::9].shape) + 0.5).astype(np.float32)
    specials = np.array([0.0, -0.0, -2.0, np.nan, np.inf, -np.inf], np.float32)
    raw[:, 3::23] = specials[r.integers(0, len(specials), raw[:, 3::23].shape)]
    pins = np.where(r.random((B, Tp)) < 0.25, r.integers(1, 128, (B, Tp)), -1) if pinned else np.full((B, Tp), -1)
    if pinned and B > 3:
        pins[3] = r.integers(1, 128, Tp)                                    # every phone pinned
    free = (pins < 1).sum(1)
    psum = np.where(pins >= 1, pins, 0).sum(1)
    total = free + psum + np.floor(r.random(B) * 127 * free).astype(np.int64)
    total[0] = free[0] + psum[0]
    total[1 % B] = 128 * free[1 % B] + psum[1 % B]
    return raw, pins if pinned else None, total


@pytest.mark.parametrize("pinned", [False, True], ids=["free", "pinned"])
@pytest.mark.parametrize("scale_kind", ["utterance", "phone"])
@pytest.mark.parametrize("Tp", [1, 7, 64, 1000, 8192])
def test_fit_kernel_equals_the_oracle(Tp, scale_kind, pinned):
    B = 64
    raw, pins, total = fit_case(B, Tp, Tp * 10 + pinned, pinned)
    r = np.random.default_rng(Tp)
    scale = (r.uniform(0.3, 3.0, B) if scale_kind == "utterance" else r.uniform(0.3, 3.0, (B, Tp))).astype(np.float32)
    scale[0] = 1.0
    if scale_kind == "phone":
        scale[5 % B] = 1.0
    # the no-total durations' sum as row 2's total: theta = 1 gives them back unchanged
    no_total = DC.fit(raw, scale, None, pins)
    if B > 2 and (pins is None or (pins[2] < 1).any()):
        total[2] = int(no_total[2].sum())
    raw_d = torch.from_numpy(raw).to(DEV)
    for tot in (None, total):
        got = ops.fit_durations(raw_d, torch.from_numpy(scale), None if tot is None else torch.from_numpy(tot),
                                None if pins is None else torch.from_numpy(pins)).cpu()
        want = no_total if tot is None else DC.fit(raw, scale, tot, pins)
        assert got.dtype == torch.int32 and torch.equal(got, want), tot is None
        if tot is not None:
            assert got.sum(1).tolist() == total.tolist()
            if B > 2 and (pins is None or (pins[2] < 1).any()):
                assert torch.equal(got[2], no_total[2])
    # a scalar scale and no scale at all
    for sc in (None, 1.75):
        got = ops.fit_durations(raw_d, sc, torch.from_numpy(total), None if pins is None else torch.from_numpy(pins))
        assert torch.equal(got.cpu(), DC.fit(raw, sc, total, pins)), sc


def test_fit_kernel_ties_and_strided_input():
    """Equal values at one level across 8192 phones (the boundary ties are settled by phone index across every thread of
    the CTA), and raw values read at a batch stride wider than Tp."""
    B, Tp = 4, 8192
    raw = np.full((B, Tp), 6.0, np.float32)
    raw[1, ::2] = 3.0
    raw[2] = 0.0
    total = np.array([Tp + 5000, Tp + Tp + 777, Tp + 3 * 127 + 5, Tp + 2 * Tp + 1])
    wide = torch.zeros(B, Tp + 3)
    wide[:, :Tp] = torch.from_numpy(raw)
    got = ops.fit_durations(wide.to(DEV)[:, :Tp], None, torch.from_numpy(total)).cpu()
    assert torch.equal(got, DC.fit(raw, None, total))
    assert got[2, :3].tolist() == [128, 128, 128] and got[2, 3].item() == 6 and got[2, 4:].eq(1).all()


def test_fit_with_scale_one_equals_infer(tts):
    tc = sources(1, 8, 37, 300)[0]
    dur, raw = tts.adm.infer(tc, return_raw=True)
    assert torch.equal(ops.fit_durations(raw), dur[..., 0])
    assert torch.equal(ops.fit_durations(raw, 1.0), dur[..., 0])


# ------------------------------------------------------------------------------ pinned decodes: identities
def free_pins(B, T):
    return torch.full((B, T), -1, dtype=torch.int32)


def some_pins(B, T, seed):
    r = np.random.default_rng(seed)
    p = np.where(r.random((B, T)) < 0.3, r.integers(1, 128, (B, T)), -1)
    p[0, 0] = 40
    p[-1, -1] = 1
    return torch.from_numpy(p).to(torch.int32)


@ENGINES
def test_all_free_pins_equal_the_unpinned_decodes(tts, engine):
    adm = tts.adm
    K, B, T = 2, 3, 18
    tcs = sources(K, B, T, 500)
    sched = torch.rand(B, T, K, generator=gen(501)) + 0.1
    with pack.engine_scope(engine):
        for _ in range(3):                                          # eager, capture, replay
            a = adm.infer(tcs[0], return_raw=True)
            b = adm.infer(tcs[0], return_raw=True, pinned=free_pins(B, T))
            assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
            for w in ([0.3, 0.7], sched):
                a = adm.infer_mix(tcs, w, return_raw=True)
                b = adm.infer_mix(tcs, w, return_raw=True, pinned=free_pins(B, T))
                for x, y in zip(a, b):
                    assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_one_hot_mix_with_pins_equals_the_plain_decode_on_the_stack(tts):
    adm = tts.adm
    K, B, T = 3, 3, 12
    tcs = sources(K, B, T, 600)
    pins = some_pins(B, T, 601)
    with graphs.disabled():
        ref_dur, ref_raw = adm.infer(torch.cat(tcs, 0), return_raw=True, pinned=pins.repeat(K, 1))
    for k in range(K):
        w = torch.zeros(K)
        w[k] = 2.0
        for _ in range(3):
            dur, raw, raw_src = adm.infer_mix(tcs, w, return_raw=True, pinned=pins)
            blk = slice(k * B, (k + 1) * B)
            assert torch.equal(dur, ref_dur[blk]) and torch.equal(raw.view(torch.int32), ref_raw[blk].view(torch.int32))
            # raw_src keeps the sources' own readouts: at pinned steps they are not the pins
            on = pins.to(DEV) >= 1
            assert torch.equal(raw_src[k][~on], ref_raw[blk][~on])
            assert not torch.equal(raw_src[k][on], raw[on])
    pd = pins.to(DEV)
    assert torch.equal(ref_dur[:B, :, 0][pd >= 1], pd[pd >= 1])


def test_new_pins_replay_without_a_new_capture(tts):
    adm = tts.adm
    B, T = 4, 10
    tc = sources(1, B, T, 700)[0]
    for _ in range(2):                                                 # warm-up, capture
        adm.infer(tc, return_raw=True, pinned=some_pins(B, T, 701))
    n_graphs, n_replayed = len(adm._graphs().cache), graphs.replayed_launches
    outs = set()
    for seed in range(702, 706):
        pins = some_pins(B, T, seed)
        got = adm.infer(tc, return_raw=True, pinned=pins)
        with graphs.disabled():
            want = adm.infer(tc, return_raw=True, pinned=pins)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), seed
        pd = pins.to(DEV)
        assert torch.equal(got[0][..., 0][pd >= 1], pd[pd >= 1])
        outs.add(tuple(got[1].flatten().tolist()))
    assert len(adm._graphs().cache) == n_graphs and graphs.replayed_launches > n_replayed
    assert len(outs) == 4


# ------------------------------------------------------------------------------ pinned decodes against fp64
@pytest.fixture(scope="module")
def fp64_pinned(weights_cpu):
    """K = 2 and K = 1 (plain) pinned decodes of B = 4, T = 20 and their fp64 restatements, computed once."""
    K, B, T = 2, 4, 20
    tcs = [torch.randn(B, T, 512, generator=gen(910 + k)).abs() for k in range(K)]
    w = np.array([[0.3, 0.7], [1.0, 0.0], [0.0, 2.0], [0.6, 0.4]], np.float32)
    pins = some_pins(B, T, 912)
    sd = DC.DM.sd64(weights_cpu("adm"))
    with torch.no_grad():
        mix = DC.adm_infer_pinned(sd, [t.double() for t in tcs], weights.ADM_CFG, w, pins, return_raw=True)[1]
        plain = DC.adm_infer_pinned(sd, [tcs[0].double()], weights.ADM_CFG, np.ones((B, 1), np.float32), pins,
                                    return_raw=True)[1]
    return tcs, w, pins, mix[..., 0], plain[..., 0]


@ENGINES
@pytest.mark.parametrize("mixed", [False, True], ids=["plain", "mix"])
def test_pinned_decode_against_the_fp64_oracle(tts, fp64_pinned, engine, mixed):
    tcs, w, pins, mix64, plain64 = fp64_pinned
    with pack.engine_scope(engine):
        if mixed:
            dur, raw, _ = tts.adm.infer_mix([t.to(DEV) for t in tcs], w, return_raw=True, pinned=pins)
        else:
            dur, raw = tts.adm.infer(tcs[0].to(DEV), return_raw=True, pinned=pins)
    raw64 = mix64 if mixed else plain64
    dur, raw = dur.cpu()[..., 0], raw.cpu().double()
    on = pins >= 1
    assert torch.equal(dur[on], pins[on]) and torch.equal(raw[on], pins[on].double())
    err = (raw - raw64)[~on].abs().max().item()
    scale = max(1.0, raw64[~on].abs().max().item())
    near = _boundary_distance(raw64) <= NEAR
    helpers.record("duration_control_vs_fp64", dict(engine=engine, mixed=mixed, max_abs=err, scale=scale))
    print(f"engine {engine} {'mix' if mixed else 'plain'}: max |raw - raw_fp64| over free phones = {err:.3g} "
          f"(scale {scale:.3g})")
    assert err <= RAW_REL * scale
    want = (raw64 + 0.5).to(torch.int32).clamp(1, 128)
    assert torch.equal(dur[~on & ~near], want[~on & ~near])


# ------------------------------------------------------------------------------ end to end
def _inputs(B=3, Tp=9):
    phone = torch.randint(0, 320, (B, Tp), generator=gen(61)).to(DEV)
    melp = (torch.randn(B, 56, 80, generator=gen(62)) * 2 - 4).to(DEV)
    pros = [(torch.randn(B, 40, 80, generator=gen(63)) * 2 - 3).to(DEV)]
    pins = torch.full((B, Tp), -1, dtype=torch.int32)
    pins[0, 2], pins[1, 0], pins[2, Tp - 1] = 40, 12, 3
    return phone, melp, pros, pins


@pytest.mark.parametrize("mode", ["plain", "duration_mix", "causal"])
def test_synthesize_fits_the_requested_lengths(tts, mode):
    phone, melp, pros, pins = _inputs()
    B = phone.shape[0]
    scale = torch.tensor([1.25, 0.8, 1.0])
    kw = dict(duration_scale=scale)
    if mode == "causal":
        kw["causal_decode"] = True
    else:
        kw["pinned_durations"] = pins
    if mode == "duration_mix":
        kw.update(prosody_mels=pros, prosody_weights=[0.5, 0.5], duration_weights=[0.3, 0.7])
    with torch.no_grad():
        tc = tts.generator.mrte.tc_latent(phone, melp)
        if mode == "plain":
            raw = tts.adm.infer(tc, return_raw=True, pinned=pins)[1]
        elif mode == "causal":
            raw = tts.adm.infer_causal(tc, return_raw=True)[1]
        else:
            raw = tts.adm.infer_mix([tc, tts.generator.mrte.tc_latent(phone, pros[0])], [0.3, 0.7], return_raw=True,
                                    pinned=pins)[1]
    base = ops.fit_durations(raw, scale, None, kw.get("pinned_durations"))
    total = (base.sum(1).cpu().double() * 1.25).round().to(torch.int64)
    out = tts.synthesize(phone, melp, total_frames=total, return_intermediates=True, **kw)
    assert out["totals"] == total.tolist()
    assert out["wav_lens"] == [256 * (t + 10) for t in total.tolist()]
    assert out["wav"].shape[-1] == 256 * (max(total.tolist()) + 10)
    want = ops.fit_durations(raw, scale, total, kw.get("pinned_durations"))
    assert torch.equal(out["dt"], want) and out["dt"].sum(1).tolist() == total.tolist()
    if mode != "causal":
        pd = pins.to(DEV)
        assert torch.equal(out["dt"][pd >= 1], pd[pd >= 1])
    # without a total: the scaled rounding; pins alone: the ADM's own (pinned) durations
    out = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    assert torch.equal(out["dt"], base) and out["totals"] == base.sum(1).tolist()
    if mode == "plain":
        out = tts.synthesize(phone, melp, pinned_durations=pins, return_intermediates=True)
        assert torch.equal(out["dt"], tts.adm.infer(tc, pinned=pins)[..., 0])
    assert B == 3


def test_stream_equals_synthesize(tts):
    phone, melp, pros, pins = _inputs()
    total = torch.tensor([70, 41, 96])
    kw = dict(duration_scale=1.1, total_frames=total, pinned_durations=pins, prosody_mels=pros,
              prosody_weights=[0.6, 0.4], duration_weights=[0.5, 0.5], sampling=Sampling(temperature=0.9, seed=5),
              keys=torch.arange(3))
    ref = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    assert ref["totals"] == total.tolist()
    for cf in (8, 200):
        chunks = list(tts.synthesize_stream(phone, melp, chunk_frames=cf, **kw))
        wav = torch.cat([c["wav"] for c in chunks], -1)
        assert torch.equal(chunks[-1]["p_codes"], ref["p_codes"]) and torch.equal(chunks[-1]["dt"], ref["dt"])
        assert chunks[-1]["wav_lens"] == ref["wav_lens"] and wav.shape == ref["wav"].shape
        assert (wav - ref["wav"]).abs().max().item() <= 1e-5, cf


def test_range_flag_rerun_keeps_the_requested_lengths(golden, weights_cpu):
    """The scaled-attention overflow of the prosody-mix range test: synthesize warns and reruns the batch on bf16x3, and
    the rerun still has the requested totals and equals a bf16x3 run."""
    g = golden("e2e")
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    phone = torch.randint(0, 320, (1, 70), generator=gen(13)).to(DEV)
    melp = g["mel_prompt"].to(DEV)
    lyr = tts.plm.plm.layers[0]
    with torch.no_grad():
        lyr.attn.w_q.weight.mul_(2.0 ** 17)
        lyr.attn.w_k.weight.mul_(2.0 ** -17)
    pins = torch.full((1, 70), -1, dtype=torch.int32)
    pins[0, 10] = 30
    kw = dict(total_frames=[600], duration_scale=0.9, pinned_durations=pins)   # 75 PLM steps: tensor-core attention
    ops.tc_overflow(torch.device(DEV))
    with pack.engine_scope(pack.ENGINE_F16X2):
        with pytest.warns(UserWarning, match="fp16 range"):
            ref = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    with pack.engine_scope(pack.ENGINE_BF16X3):
        want = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    assert ref["totals"] == [600] and want["totals"] == [600]
    assert torch.equal(ref["dt"], want["dt"]) and ref["dt"][0, 10].item() == 30
    assert torch.equal(ref["p_codes"], want["p_codes"]) and torch.equal(ref["wav"], want["wav"])


def test_synthesize_many_with_a_scalar_scale(tts):
    phone, melp, _, _ = _inputs()
    items = [(phone[i], melp[i]) for i in range(3)]
    slow = tts.synthesize_many(items, duration_scale=1.5)
    ref = tts.synthesize(phone, melp, duration_scale=1.5, return_intermediates=True)
    assert [w.shape[-1] for w in slow] == ref["wav_lens"]


def test_rejections(tts):
    phone, melp, pros, pins = _inputs()
    forced = torch.full((3, 9), 4, dtype=torch.int32, device=DEV)
    for kw in (dict(forced_durations=forced, duration_scale=1.2), dict(forced_durations=forced, total_frames=[9] * 3),
               dict(forced_durations=forced, pinned_durations=pins), dict(causal_decode=True, pinned_durations=pins),
               dict(total_frames=[8, 9, 9]), dict(total_frames=[9, 9, 128 * 9 + 1]),
               dict(total_frames=[9, 9, 9], pinned_durations=pins), dict(duration_scale=torch.ones(3, 8)),
               dict(duration_scale=-1.0), dict(pinned_durations=pins.to(torch.float32))):
        n0 = ops.launch_count()
        with pytest.raises(L.MttsError):
            tts.synthesize(phone, melp, **kw)
        assert ops.launch_count() == n0, kw                           # rejected before any device work
    with pytest.raises(L.MttsError):
        tts.adm.infer(torch.zeros(2, 4, 512, device=DEV), pinned=torch.zeros(2, 4, dtype=torch.int32))
    with pytest.raises(L.MttsError):
        ops.fit_durations(torch.zeros(2, 8193, device=DEV))
