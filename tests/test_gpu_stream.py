"""Streamed synthesis on the GPU: the resumable PLM decode against ``MegaPLM.infer``, ``Megatts.synthesize_stream`` against
``synthesize`` and the CPU oracle, and the stream's fp16 range-flag policy."""
import random

import pytest
import torch

import helpers
from megatts2_b200 import graphs, ops, pack
from megatts2_b200.sampling import Sampling
from oracle import ref_megatts2 as R
from oracle import weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda"


def gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


@pytest.fixture(scope="module")
def tts(weights_cpu):
    return helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)


def _splits(T, rng):
    """split points of [0, T): one range, one-step ranges, and a random split"""
    cuts = sorted(rng.sample(range(1, T), min(T - 1, 3))) if T > 1 else []
    return [[0, T], list(range(T + 1)), [0] + cuts + [T]]


SAMPLINGS = [None, Sampling(temperature=0.8, top_k=20, seed=5), Sampling(temperature=1.3, top_p=0.9, seed=2 ** 63 + 11)]


@pytest.mark.parametrize("B,T", [(1, 1), (1, 9), (5, 9), (5, 70), (1, 70)])
@pytest.mark.parametrize("smp", range(len(SAMPLINGS)))
def test_plm_ranges_equal_infer(tts, B, T, smp):
    """Any split of [0, T) into ranges gives infer's codes and logits bit for bit, eager and through replayed graphs."""
    plm = tts.plm
    sampling = SAMPLINGS[smp]
    tc = torch.randn(B, T, plm.tc_latent_dim, generator=gen(100 + B * T)).to(DEV)
    keys = torch.arange(7, 7 + B, dtype=torch.int64)
    kw = {} if sampling is None else dict(sampling=sampling, keys=keys)
    with graphs.disabled():
        ref_codes, ref_logits = plm.infer(tc, return_logits=True, **kw)
    rng = random.Random(T * 31 + B + smp)
    for graphed in (False, True):
        for cuts in _splits(T, rng):
            for rep in range(3 if graphed else 1):            # warm-up, capture, replay
                dec = plm.begin_decode(tc, **kw)
                codes, logits = [], []
                for t0, t1 in zip(cuts, cuts[1:]):
                    if graphed:
                        c, lg = plm.decode_until(dec, t1, return_logits=True)
                    else:
                        with graphs.disabled():
                            c, lg = plm.decode_until(dec, t1, return_logits=True)
                    assert c.shape == (B, t1 - t0)
                    codes.append(c)
                    logits.append(lg)
                assert dec.t == T
                assert torch.equal(torch.cat(codes, 1), ref_codes), (graphed, cuts, rep)
                assert torch.equal(torch.cat(logits, 1), ref_logits), (graphed, cuts, rep)
                assert torch.equal(dec.codes, ref_codes)
    with pytest.raises(Exception):
        plm.decode_until(plm.begin_decode(tc), T + 1)


def _run_stream(tts, *args, **kw):
    chunks = list(tts.synthesize_stream(*args, **kw))
    assert chunks and chunks[-1]["last"] and not any(c["last"] for c in chunks[:-1])
    off = 0
    for c in chunks:
        assert c["offset"] == off
        off += c["wav"].shape[-1]
    wav = torch.cat([c["wav"] for c in chunks], -1)
    valid = [sum(c["valid"][b] for c in chunks) for b in range(wav.shape[0])]
    return chunks, wav, valid


def _inputs(kind, durations, tts):
    if kind == "golden":
        from conftest import load_golden
        g = load_golden("e2e")
        phone, melp = g["phone"].to(DEV), g["mel_prompt"].to(DEV)
        forced = g["dt_used"].to(DEV)
    else:
        phone = torch.randint(0, 320, (3, 9), generator=gen(61)).to(DEV)
        melp = (torch.randn(3, 56, 80, generator=gen(62)) * 2 - 4).to(DEV)
        forced = (torch.full((3, 9), 4, dtype=torch.int32) if durations == "equal" else
                  torch.randint(1, 7, (3, 9), generator=gen(63), dtype=torch.int32)).to(DEV)
    return phone, melp, (None if durations == "adm" else forced)


CASES = [(k, d) for k in ("golden", "batch3") for d in ("equal", "ragged", "adm") if not (k == "golden" and d == "ragged")]


@pytest.mark.parametrize("kind,durations", CASES)
@pytest.mark.parametrize("prompt", [False, True])
@pytest.mark.parametrize("sampled", [False, True])
def test_stream_equals_synthesize(tts, kind, durations, prompt, sampled):
    phone, melp, forced = _inputs(kind, durations, tts)
    kw = dict(forced_durations=forced, prompt_mels=melp if prompt else None)
    if sampled:
        kw.update(sampling=Sampling(temperature=0.9, top_k=50, seed=17), keys=torch.arange(3, 3 + phone.shape[0]))
    ref = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    if durations == "ragged":
        assert len(set(ref["totals"])) > 1
    Lmax = max(ref["totals"])
    for cf in (8, 64, Lmax + 100):
        chunks, wav, valid = _run_stream(tts, phone, melp, chunk_frames=cf, **kw)
        last = chunks[-1]
        assert torch.equal(last["p_codes"], ref["p_codes"]) and torch.equal(last["dt"], ref["dt"])
        assert last["wav_lens"] == ref["wav_lens"] and valid == ref["wav_lens"]
        assert wav.shape == ref["wav"].shape
        err = (wav - ref["wav"]).abs().max().item()
        helpers.record("stream_vs_synthesize", dict(kind=kind, durations=durations, prompt=prompt, sampled=sampled,
                                                    chunk_frames=cf, totals=ref["totals"], max_abs=err,
                                                    bit_identical=bool(torch.equal(wav, ref["wav"]))))
        assert err <= 1e-5, (cf, err)
        if prompt:
            assert torch.equal(chunks[0]["wav"], ref["wav"][..., :chunks[0]["wav"].shape[-1]])
        for b, n in enumerate(ref["wav_lens"]):                  # zeros past a shorter utterance's end
            assert float(wav[b, :, n:].abs().max()) == 0.0 if n < wav.shape[-1] else True


def test_stream_equals_the_oracle(weights_cpu, tts):
    """One utterance against the CPU oracle, within the bars of test_e2e_vs_oracle_batched."""
    phone = torch.randint(0, 320, (1, 9), generator=gen(71))
    melp = torch.randn(1, 72, 80, generator=gen(72)) * 2 - 4              # (B, frames, 80), as both sides take it
    forced = torch.randint(2, 9, (1, 9), generator=gen(73), dtype=torch.int32)
    cfgs = (weights.G_CFG, weights.PLM_CFG, weights.ADM_CFG, weights.HIFIGAN_CFG)
    ref = R.synthesize(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), phone,
                       melp, cfgs, forced_durations=forced)
    chunks, wav, valid = _run_stream(tts, phone.to(DEV), melp.to(DEV), forced_durations=forced.to(DEV), chunk_frames=16)
    last = chunks[-1]
    t = int(forced.sum())
    assert len(chunks) > 2
    assert torch.equal(last["dt"].cpu(), ref["dt"]) and torch.equal(last["p_codes"].cpu(), ref["p_codes"])
    assert (last["mel"][:, :t].cpu() - ref["mel"].transpose(1, 2)).abs().mean().item() < 1e-4
    assert (wav.cpu() - ref["wav"]).abs().max().item() < 1e-3


def test_stream_range_flag_restarts_on_bf16x3(golden, weights_cpu):
    """The scaled-attention overflow of test_synthesize_attention_overflow_reruns_finite_on_bf16x3.  In one chunk it is
    raised before anything is yielded, so the stream warns, restarts on bf16x3 and equals synthesize's rerun.  In chunks of
    64 frames it is raised after the first chunk: the stream warns and finishes on bf16x3, with finite samples."""
    dev = torch.device(DEV)
    g = golden("e2e")
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    phone = torch.randint(0, 320, (1, 70), generator=gen(13)).to(DEV)
    dur = torch.full((1, 70), 8, dtype=torch.int32, device=DEV)
    lyr = tts.plm.plm.layers[0]
    with torch.no_grad():
        lyr.attn.w_q.weight.mul_(2.0 ** 17)
        lyr.attn.w_k.weight.mul_(2.0 ** -17)
    ops.tc_overflow(dev)
    with pack.engine_scope(pack.ENGINE_F16X2):
        with pytest.warns(UserWarning, match="fp16 range"):
            ref = tts.synthesize(phone, g["mel_prompt"].to(DEV), forced_durations=dur, return_intermediates=True)
        with pytest.warns(UserWarning, match="restarting this stream on the bf16x3 engine"):
            chunks, wav, _ = _run_stream(tts, phone, g["mel_prompt"].to(DEV), forced_durations=dur, chunk_frames=1000)
        with pytest.warns(UserWarning, match="finishing this stream on the bf16x3 engine"):
            late, wav_late, _ = _run_stream(tts, phone, g["mel_prompt"].to(DEV), forced_durations=dur, chunk_frames=64)
    assert len(chunks) == 1 and bool(torch.isfinite(wav).all())
    assert torch.equal(chunks[-1]["p_codes"], ref["p_codes"])
    assert wav.shape == ref["wav"].shape and (wav - ref["wav"]).abs().max().item() <= 1e-5
    assert len(late) > 1 and wav_late.shape == ref["wav"].shape and bool(torch.isfinite(wav_late).all())


def test_stream_rejects_unsupported_arguments(tts):
    phone = torch.randint(0, 320, (1, 4), generator=gen(81)).to(DEV)
    melp = torch.randn(1, 40, 80, generator=gen(82)).to(DEV)
    for kw in (dict(causal_decode=True), dict(overlap_prompt=True), dict(chunk_frames=0)):
        with pytest.raises(Exception):
            next(iter(tts.synthesize_stream(phone, melp, **kw)))
