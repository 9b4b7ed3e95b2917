"""GPU: timbre interpolation.  The mix + LayerNorm kernel (csrc/ops.cu, mix_layernorm_kernel) against fp64 and against
layernorm, MRTE.tc_latent_mix against the fp64 restatement (tests/ref_timbre_mix.py) and against tc_latent, and
Megatts.synthesize / synthesize_stream with timbre_mels.

Bars: the kernel within KERNEL_TOL (1 + |fp64 value|) of the fp64 mix + LayerNorm + ReLU of the same fp32 rows; the
latent within MRTE_MAX / MRTE_MEAN of the fp64 restatement (the bars test_gpu_parity allows tc_latent against its fp64
golden); one-hot rows, schedules that repeat one row, and everything the timbre mix must leave alone, bit for bit."""
import numpy as np
import pytest
import torch

import helpers
import ref_duration_mix as DM
import ref_timbre_mix as RT
from megatts2_b200 import _lib as L
from megatts2_b200 import ops, pack
from megatts2_b200.models.megatts2 import PLMContext
from megatts2_b200.sampling import Sampling
from oracle import weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda"
KERNEL_TOL = 2e-5
MRTE_MAX, MRTE_MEAN = 2e-4, 2e-5
ENGINES = pytest.mark.parametrize("engine", [pack.ENGINE_F16X2, pack.ENGINE_BF16X3, pack.ENGINE_FFMA],
                                  ids=["f16x2", "bf16x3", "ffma"])


def gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def tts(weights_cpu):
    return helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)


def _weights(shape, K, B, T, seed):
    """Random weights of `shape` with zeros (whole sources for (K,), rows' entries otherwise) and one-hot rows."""
    r = np.random.default_rng(seed)
    if shape == "K":
        w = r.random(K).astype(np.float32) + 0.05
        if K > 1:
            w[K // 2] = 0.0
        return w
    w = r.random((B, K) if shape == "BK" else (B, T, K)).astype(np.float32) + 0.05
    flat = w.reshape(-1, K)
    if K > 1:
        flat[::3, 0] = 0.0
        flat[1::4] = np.eye(K, dtype=np.float32)[np.arange(len(flat[1::4])) % K] * 3.0
    return w


def _poison(ys, w):
    """ys (K, B, T, C) with every element of a zero-weight source row set to NaN or inf (never read by the kernel)."""
    K, B, T, _ = ys.shape
    wr = RT.weight_rows(w, K, B, T)
    ys = ys.clone()
    for k in range(K):
        off = wr[..., k] == 0
        ys[k][off] = float("nan") if k % 2 else float("inf")
    return ys


# ------------------------------------------------------------------------------ kernel level
@pytest.mark.parametrize("shape", ["K", "BK", "BTK"])
@pytest.mark.parametrize("C", [384, 512, 768, 1024])
@pytest.mark.parametrize("K", [1, 2, 8])
def test_mix_layernorm_against_fp64(K, C, shape):
    B, T = 3, 37
    ys = torch.randn(K, B, T, C, generator=gen(K * 7 + C)) * (1 + torch.arange(K).view(K, 1, 1, 1))
    gamma, beta = torch.randn(C, generator=gen(C)), torch.randn(C, generator=gen(C + 1)) * 0.1
    w = _weights(shape, K, B, T, K + C)
    want = RT.mix_layernorm(ys, w, gamma, beta)
    clean = ops.mix_layernorm(ys.to(DEV), torch.from_numpy(w).to(DEV), gamma.to(DEV), beta.to(DEV),
                              post_act=L.ACT_RELU).cpu()
    err = ((clean.double() - want).abs() / (1 + want.abs())).max().item()
    assert err <= KERNEL_TOL, err
    got = ops.mix_layernorm(_poison(ys, w).to(DEV), torch.from_numpy(w).to(DEV), gamma.to(DEV), beta.to(DEV),
                            post_act=L.ACT_RELU).cpu()
    assert torch.isfinite(got).all() and torch.equal(got, clean)


@pytest.mark.parametrize("act", [L.ACT_RELU, L.ACT_NONE])
@pytest.mark.parametrize("C", [384, 512, 768, 1024])
def test_one_hot_rows_equal_layernorm(C, act):
    B, T, K = 4, 29, 5
    ys = torch.randn(K, B, T, C, generator=gen(C + 5)).to(DEV) * 3 - 1
    gamma, beta = torch.randn(C, generator=gen(C)).to(DEV), torch.randn(C, generator=gen(C + 1)).to(DEV)
    src = torch.randint(0, K, (B, T), generator=gen(C + 7))
    w = torch.nn.functional.one_hot(src, K).float() * (torch.rand(B, T, 1, generator=gen(C + 8)) * 5 + 1e-3)
    got = ops.mix_layernorm(_poison(ys.cpu(), w).to(DEV), w.to(DEV), gamma, beta, post_act=act)
    for k in range(K):
        ln = ops.layernorm(ys[k], gamma, beta, post_act=act)
        m = (src == k).to(DEV)
        assert torch.equal(got[m], ln[m]), k


def test_zero_weight_rows_and_strided_sources():
    """A source view with a row stride above C and a K stride between separate buffers' slots reads the right rows."""
    K, B, T, C = 3, 2, 9, 512
    big = torch.randn(K, B, T, C + 64, generator=gen(1)).to(DEV)
    ys = big[..., :C]
    gamma, beta = torch.ones(C, device=DEV), torch.zeros(C, device=DEV)
    w = torch.tensor([[0.2, 0.3, 0.5], [0.0, 0.0, 1.0]], device=DEV)
    got = ops.mix_layernorm(ys, w, gamma, beta)
    want = ops.mix_layernorm(ys.contiguous(), w, gamma, beta)
    assert torch.equal(got, want)
    assert torch.equal(got[1], ops.layernorm(ys[2, 1], gamma, beta))


# ------------------------------------------------------------------------------ tc_latent_mix
def _mrte_inputs(B=2, Tp=23):
    phone = torch.randint(0, 320, (B, Tp), generator=gen(31))
    mels = [torch.randn(B, Tm, 80, generator=gen(32 + i)) * s - o
            for i, (Tm, s, o) in enumerate([(56, 2.0, 4.0), (40, 1.5, 3.0), (72, 2.5, 5.0)])]
    return phone, mels


@pytest.fixture(scope="module")
def fp64_case(weights_cpu):
    phone, mels = _mrte_inputs()
    w = (np.random.default_rng(5).random((2, 23, 3)) + 0.05).astype(np.float32)
    w[0, :5] = [0.0, 1.0, 0.0]
    sd = DM.sd64(weights_cpu("g")).sub("mrte")
    with torch.no_grad():
        want = RT.tc_latent_mix(sd, phone, [m.double() for m in mels], w, weights.G_CFG)
    return phone, mels, w, want


@ENGINES
def test_tc_latent_mix_against_fp64(tts, fp64_case, engine):
    phone, mels, w, want = fp64_case
    with pack.engine_scope(engine), torch.no_grad():
        got = tts.generator.mrte.tc_latent_mix(phone.to(DEV), [m.to(DEV) for m in mels], w).cpu()
    err = (got.double() - want).abs()
    print(f"engine {engine}: tc_latent_mix vs fp64 max {err.max().item():.3g} mean {err.mean().item():.3g}")
    helpers.record("timbre_mix_vs_fp64", dict(engine=engine, max_abs=err.max().item(), mean_abs=err.mean().item()))
    assert err.max().item() < MRTE_MAX and err.mean().item() < MRTE_MEAN


@ENGINES
def test_tc_latent_mix_one_hot_and_schedules(tts, engine):
    phone, mels = _mrte_inputs()
    phone, mels = phone.to(DEV), [m.to(DEV) for m in mels]
    mrte = tts.generator.mrte
    with pack.engine_scope(engine), torch.no_grad():
        lats = [mrte.tc_latent(phone, m) for m in mels]
        for k in range(3):
            one = [0.0] * 3
            one[k] = 0.7
            assert torch.equal(mrte.tc_latent_mix(phone, mels, one), lats[k]), k
        src = torch.randint(0, 3, (2, 23), generator=gen(9))
        src[:, :4], src[:, 4:9] = 0, 2                        # runs of phones on one source, then switches
        sched = torch.nn.functional.one_hot(src, 3).float() * 2.5
        got = mrte.tc_latent_mix(phone, mels, sched)
        for k in range(3):
            m = (src == k).to(DEV)
            assert torch.equal(got[m], lats[k][m]), k
        row = torch.tensor([[0.2, 0.5, 0.3], [0.0, 0.6, 0.4]])
        assert torch.equal(mrte.tc_latent_mix(phone, mels, row[:, None].expand(2, 23, 3)),
                           mrte.tc_latent_mix(phone, mels, row))


# ------------------------------------------------------------------------------ synthesis
def _e2e_inputs(durations="equal", B=3, Tp=9):
    phone = torch.randint(0, 320, (B, Tp), generator=gen(61)).to(DEV)
    melp = (torch.randn(B, 56, 80, generator=gen(62)) * 2 - 4).to(DEV)
    timbre = [(torch.randn(B, 40, 80, generator=gen(63)) * 2 - 3).to(DEV),
              (torch.randn(B, 72, 80, generator=gen(64)) * 1.5 - 5).to(DEV)]
    forced = (torch.full((B, Tp), 4, dtype=torch.int32) if durations == "equal" else
              torch.randint(1, 7, (B, Tp), generator=gen(65), dtype=torch.int32)).to(DEV)
    return phone, melp, timbre, (None if durations == "adm" else forced)


W3 = torch.tensor([[0.5, 0.25, 0.25], [0.0, 1.0, 0.0], [0.1, 0.0, 0.9]])
SMP = dict(sampling=Sampling(temperature=0.9, top_k=50, seed=17), keys=torch.arange(3))


def _compose(tts, blend, d, p_codes):
    """The mel decoder and the vocoder on ``blend`` length-regulated by d, composed by hand as synthesize composes them:
    one batch when every utterance has the same frame total, else one per group of equal totals (zeros past a total)."""
    with torch.no_grad():
        tce, totals = ops.length_regulate(blend, d, return_host_totals=True)
        B, Lmax = tce.shape[0], tce.shape[1]
        if all(t == Lmax for t in totals):
            mel = tts.generator.decode_mel_cl(tce, p_codes)
            return mel, tts.hifi_gan.decode_batch_cl(mel)
        mel = torch.zeros(B, Lmax, 80, device=DEV)
        wav = torch.zeros(B, 1, 256 * (Lmax + 10), device=DEV)
        for Lg in sorted(set(totals) - {0}):
            idx = [i for i, t in enumerate(totals) if t == Lg]
            mg = tts.generator.decode_mel_cl(tce[idx, :Lg].contiguous(), p_codes[idx, :(Lg + 7) // 8].contiguous())
            wg = tts.hifi_gan.decode_batch_cl(mg)
            mel[idx, :Lg] = mg
            wav[idx, :, :wg.shape[-1]] = wg
        return mel, wav


@ENGINES
@pytest.mark.parametrize("durations", ["adm", "equal"])
def test_synthesize_blend(tts, engine, durations):
    phone, melp, timbre, forced = _e2e_inputs(durations)
    with pack.engine_scope(engine):
        base = tts.synthesize(phone, melp, forced_durations=forced, return_intermediates=True, **SMP)
        zero = tts.synthesize(phone, melp, forced_durations=forced, return_intermediates=True, timbre_mels=timbre,
                              timbre_weights=[2.0, 0.0, 0.0], **SMP)
        mixed = tts.synthesize(phone, melp, forced_durations=forced, return_intermediates=True, timbre_mels=timbre,
                               timbre_weights=W3, **SMP)
        with torch.no_grad():
            want_blend = tts.generator.mrte.tc_latent_mix(phone, [melp] + timbre, W3)
            one_k = tts.generator.mrte.tc_latent(phone, timbre[1])
        onehot = tts.synthesize(phone, melp, forced_durations=forced, return_intermediates=True, timbre_mels=timbre,
                                timbre_weights=[0.0, 0.0, 1.0], **SMP)
        d = base["dt"] if forced is None else forced
        want_mel, want_wav = _compose(tts, one_k, d, base["p_codes"])
        mix_mel, mix_wav = _compose(tts, want_blend, d, base["p_codes"])
    for out in (zero, mixed, onehot):
        for k in ("dt", "p_codes", "tc_latent", "tc_latent_expand"):
            assert torch.equal(out[k], base[k]), k
    assert torch.equal(zero["mel"], base["mel"]) and torch.equal(zero["wav"], base["wav"])
    assert torch.equal(zero["timbre_latent"], base["tc_latent"])
    assert torch.equal(mixed["timbre_latent"], want_blend)
    assert torch.equal(mixed["mel"], mix_mel) and torch.equal(mixed["wav"], mix_wav)
    assert not torch.equal(mixed["mel"], base["mel"])
    assert torch.equal(onehot["mel"], want_mel) and torch.equal(onehot["wav"], want_wav)


@ENGINES
def test_ragged_totals_match_per_group_composition(tts, engine):
    phone, melp, timbre, forced = _e2e_inputs("ragged")
    with pack.engine_scope(engine):
        out = tts.synthesize(phone, melp, forced_durations=forced, return_intermediates=True, timbre_mels=timbre,
                             timbre_weights=W3)
        base = tts.synthesize(phone, melp, forced_durations=forced, return_intermediates=True)
        assert len(set(out["totals"])) > 1
        assert torch.equal(out["p_codes"], base["p_codes"])
        mel, wav = _compose(tts, out["timbre_latent"], forced, out["p_codes"])
    assert torch.equal(out["mel"], mel) and torch.equal(out["wav"], wav)


@ENGINES
def test_causal_decode_and_plm_context_combine(tts, engine):
    phone, melp, timbre, forced = _e2e_inputs("adm")
    ctx = PLMContext(torch.rand(1, 6, 512, generator=gen(70)).to(DEV), torch.randint(0, 1024, (1, 6), generator=gen(71)).to(DEV))
    sched = torch.rand(3, 9, 3, generator=gen(72)) + 0.05
    with pack.engine_scope(engine):
        for kw in (dict(causal_decode=True), dict(plm_context=ctx), dict(causal_decode=True, plm_context=ctx)):
            base = tts.synthesize(phone, melp, return_intermediates=True, **kw)
            out = tts.synthesize(phone, melp, return_intermediates=True, timbre_mels=timbre, timbre_weights=sched, **kw)
            with torch.no_grad():
                blend = tts.generator.mrte.tc_latent_mix(phone, [melp] + timbre, sched)
            mel, wav = _compose(tts, blend, base["dt"], base["p_codes"])
            assert torch.equal(out["dt"], base["dt"]) and torch.equal(out["p_codes"], base["p_codes"]), kw
            assert torch.equal(out["timbre_latent"], blend) and torch.equal(out["wav"], wav), kw


def test_full_blend_with_shared_prompts(tts):
    """The README's recipe: one prompt list and one weight set for all three mixes.  The prosody and duration mixes
    compute what they compute without the timbre mix, and the timbre latent is tc_latent_mix's."""
    phone, melp, timbre, _ = _e2e_inputs("adm")
    w = torch.rand(3, 9, 3, generator=gen(81)) + 0.05
    kw = dict(prosody_mels=timbre, prosody_weights=w, duration_weights=w, **SMP)
    base = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    out = tts.synthesize(phone, melp, return_intermediates=True, timbre_mels=timbre, timbre_weights=w,
                         total_frames=base["totals"], **kw)
    ref = tts.synthesize(phone, melp, return_intermediates=True, total_frames=base["totals"], **kw)
    with torch.no_grad():
        blend = tts.generator.mrte.tc_latent_mix(phone, [melp] + timbre, w)
    for k in ("dt", "p_codes", "tc_latent", "tc8"):
        assert torch.equal(out[k], ref[k]), k
    assert torch.equal(out["timbre_latent"], blend)
    mel, wav = _compose(tts, blend, out["dt"], out["p_codes"])
    assert torch.equal(out["mel"], mel) and torch.equal(out["wav"], wav)


def _run_stream(tts, *args, **kw):
    chunks = list(tts.synthesize_stream(*args, **kw))
    assert chunks[-1]["last"]
    return chunks, torch.cat([c["wav"] for c in chunks], -1)


@pytest.mark.parametrize("durations", ["equal", "ragged"])
def test_stream_equals_synthesize(tts, durations):
    phone, melp, timbre, forced = _e2e_inputs(durations)
    kw = dict(forced_durations=forced, prompt_mels=melp, timbre_mels=timbre, timbre_weights=torch.rand(3, 9, 3) + 0.05,
              **SMP)
    ref = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    for cf in (8, max(ref["totals"]) + 100):
        chunks, wav = _run_stream(tts, phone, melp, chunk_frames=cf, **kw)
        assert torch.equal(chunks[-1]["p_codes"], ref["p_codes"])
        assert wav.shape == ref["wav"].shape
        err = (wav - ref["wav"]).abs().max().item()
        assert err <= 1e-5, (cf, err)


def test_range_flag_reruns_on_bf16x3(golden, weights_cpu):
    """An fp16-range overflow in the prosody LM under f16x2, with a timbre mix: synthesize warns and reruns on bf16x3, and
    gives the bf16x3 run's blend, codes and waveform."""
    g = golden("e2e")
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    phone = torch.randint(0, 320, (1, 70), generator=gen(13)).to(DEV)
    dur = torch.full((1, 70), 8, dtype=torch.int32, device=DEV)
    melp = g["mel_prompt"].to(DEV)
    timbre = [(torch.randn(1, 64, 80, generator=gen(14)) * 2 - 4).to(DEV)]
    lyr = tts.plm.plm.layers[0]
    with torch.no_grad():
        lyr.attn.w_q.weight.mul_(2.0 ** 17)
        lyr.attn.w_k.weight.mul_(2.0 ** -17)
    kw = dict(forced_durations=dur, timbre_mels=timbre, timbre_weights=[0.3, 0.7])
    ops.tc_overflow(torch.device(DEV))
    with pack.engine_scope(pack.ENGINE_F16X2):
        with pytest.warns(UserWarning, match="fp16 range"):
            ref = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    with pack.engine_scope(pack.ENGINE_BF16X3):
        want = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    for k in ("timbre_latent", "p_codes", "mel", "wav"):
        assert torch.equal(ref[k], want[k]), k


def test_rejected_on_the_device_path(tts):
    phone, melp, timbre, forced = _e2e_inputs("equal")
    for kw in (dict(timbre_weights=[1, 1]), dict(timbre_weights=[1, -1, 1]), dict(timbre_weights=[0, 0, 0]),
               dict(timbre_weights=torch.ones(3, 8, 3))):
        with pytest.raises(L.MttsError, match="timbre_weights"):
            tts.synthesize(phone, melp, forced_durations=forced, timbre_mels=timbre, **kw)
    with pytest.raises(L.MttsError, match="timbre_mels"):
        tts.synthesize(phone, melp, timbre_mels=[timbre[0][:2]], timbre_weights=[1, 1])
