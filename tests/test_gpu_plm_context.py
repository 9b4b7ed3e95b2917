"""GPU: the prosody LM's in-context decode (include/megatts2_b200.h, in-context prompting).  MegaPLM.infer / infer_causal with
a context against the restatement (tests/ref_plm_context.py), its bit-for-bit identities, the causal prefill, sampling, and
Megatts.synthesize / synthesize_stream with plm_context.

Bars: step logits within test_plm_golden's 2e-3 of the restatement evaluated on the device's own code prefix, and greedy
picks equal its argmax except on rows whose two best fp32 logits are within NEAR (relative, floor 1); the range, Bc, P = 0
and replay identities bit for bit; the stream within the stream tests' 1e-5."""
import ctypes as C
import random

import pytest
import torch

import helpers
import ref_plm_context as PC
from megatts2_b200 import _lib as L
from megatts2_b200 import graphs, ops, pack
from megatts2_b200.models.megatts2 import PLMContext
from megatts2_b200.sampling import Sampling
from oracle import ref_megatts2 as R
from oracle import ref_sampling as RS
from oracle import weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = "cuda"
CFG = weights.PLM_CFG
NEAR = 1e-5
TOL = 2e-3
PS = [1, 7, 63, 64, 65, 200]
TS = [1, 9, 40]
BBC = [(1, 1), (3, 1), (3, 3)]            # (B, Bc); at B = 1, Bc = 1 is Bc = B
CHECK_STEPS = (0, 8, 39)                  # the steps compared with the restatement (the largest T's first, middle, last)


def gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def tts(weights_cpu):
    return helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)


def case_inputs(P, B, Bc):
    """Context (Bc, P) and a target latent (B, 40, 512) on the host; shorter targets are its prefixes."""
    s = 1000 * P + 10 * B + Bc
    ctx_tc = torch.randn(Bc, P, 512, generator=gen(s)).abs()
    ctx_codes = torch.randint(0, CFG["vq_bins"], (Bc, P), generator=gen(s + 1))
    tc = torch.randn(B, max(TS), 512, generator=gen(s + 2)).abs()
    return ctx_tc, ctx_codes, tc


def context(ctx_tc, ctx_codes):
    return PLMContext(ctx_tc.to(DEV), ctx_codes.to(DEV))


def near_tie(row):
    top2 = torch.topk(row.double(), 2).values
    return (top2[0] - top2[1]).item() / max(1.0, abs(top2[0].item())) <= NEAR


_ORACLE = {}      # restatement logits, keyed by the case and the device's code prefix (shared by the engines)


def oracle_step(sd, key, lat, hist, j, P):
    k = ("step", key, j, hist[:, :P + j + 1].numpy().tobytes())
    if k not in _ORACLE:
        _ORACLE[k] = R.plm_step_logits(R.SD(sd), lat, hist[:, :P + j + 1], CFG)
    return _ORACLE[k]


def oracle_causal(sd, key, ctx_tc, ctx_codes, tc, codes):
    k = ("causal", key, tc.shape[1], codes.numpy().tobytes())
    if k not in _ORACLE:
        _ORACLE[k] = PC.causal_logits_on(sd, ctx_tc, ctx_codes, tc, codes, CFG)
    return _ORACLE[k]


ENGINES = {"f16x2": pack.ENGINE_F16X2, "bf16x3": pack.ENGINE_BF16X3, "ffma": pack.ENGINE_FFMA}


@pytest.mark.parametrize("causal,engine", [(False, "f16x2"), (False, "bf16x3"), (False, "ffma"), (True, "f16x2"),
                                           (True, "bf16x3")])
def test_context_decode_against_the_restatement(weights_cpu, tts, causal, engine):
    sd, plm = weights_cpu("plm"), tts.plm
    worst, picks, ties = 0.0, 0, 0
    with pack.engine_scope(ENGINES[engine]):
        for P in PS:
            for B, Bc in BBC:
                ctx_tc, ctx_codes, tc_all = case_inputs(P, B, Bc)
                ctx = context(ctx_tc, ctx_codes)
                for T in TS:
                    tc = tc_all[:, :T]
                    dec = plm.infer_causal if causal else plm.infer
                    codes, logits = dec(tc.to(DEV), return_logits=True, context=ctx)
                    codes, logits = codes.cpu(), logits.cpu()
                    assert codes.shape == (B, T) and logits.shape == (B, T, CFG["vq_bins"])
                    key = (P, B, Bc)
                    if causal:
                        want = oracle_causal(sd, key, ctx_tc, ctx_codes, tc, codes)
                        steps = range(T)
                    else:
                        lat, hist = PC.concat(ctx_tc, ctx_codes, tc, CFG["vq_bins"])
                        hist = torch.cat([hist, codes], 1)
                        steps = [j for j in CHECK_STEPS if j < T]
                    for j in steps:
                        ref = want[:, j] if causal else oracle_step(sd, key, lat, hist, j, P)
                        err = (logits[:, j] - ref).abs().max().item()
                        worst = max(worst, err)
                        assert err <= TOL, (P, B, Bc, T, j, err)
                        for b in range(B):
                            picks += 1
                            if int(codes[b, j]) != int(ref[b].argmax()):
                                assert near_tie(ref[b]), (P, B, Bc, T, j, b)
                                ties += 1
                            assert int(codes[b, j]) == int(logits[b, j].argmax())      # greedy on its own logits
    print(f"{'causal' if causal else 'non-causal'} {engine}: max |logits - restatement| = {worst:.3g}, "
          f"{ties} of {picks} picks on near-ties")
    helpers.record("plm_context_logits", dict(causal=causal, engine=engine, max_abs=worst, picks=picks, ties=ties))


def test_f16_engine_runs(tts):
    """The half-precision engine decodes with a context; its id agreement with f16x2 is reported, not asserted."""
    plm = tts.plm
    ctx_tc, ctx_codes, tc = case_inputs(64, 3, 1)
    ctx = context(ctx_tc, ctx_codes)
    with pack.engine_scope(pack.ENGINE_F16):
        c16, l16 = plm.infer(tc.to(DEV), return_logits=True, context=ctx)
        k16, kl16 = plm.infer_causal(tc.to(DEV), return_logits=True, context=ctx)
    with pack.engine_scope(pack.ENGINE_F16X2):
        ref = plm.infer(tc.to(DEV), context=ctx)
        kref = plm.infer_causal(tc.to(DEV), context=ctx)
    assert torch.isfinite(l16).all() and torch.isfinite(kl16).all()
    agree, kagree = (c16 == ref).float().mean().item(), (k16 == kref).float().mean().item()
    print(f"f16 engine: id agreement with f16x2 {agree:.3f} (non-causal), {kagree:.3f} (causal)")
    helpers.record("plm_context_f16_agreement", dict(non_causal=agree, causal=kagree))


# ------------------------------------------------------------------------------ bit-for-bit identities
@pytest.mark.parametrize("P,B,Bc", [(7, 3, 1), (65, 3, 3), (200, 1, 1)])
def test_context_decode_is_the_range_driver_on_the_concatenation(tts, P, B, Bc):
    """The context decode equals mtts_plm_infer_range_f32 over a materialised cat(ctx_tc, tc) with the state's columns 1..P
    prefilled with the context codes, run over steps [P, P+T)."""
    plm, T = tts.plm, 9
    ctx_tc, ctx_codes, tc = case_inputs(P, B, Bc)
    tc = tc[:, :T].to(DEV)
    with graphs.disabled():
        codes, logits = plm.infer(tc, return_logits=True, context=context(ctx_tc, ctx_codes))
    N, V = P + T, plm.vq_bins
    cat = torch.cat([ctx_tc.to(DEV).expand(B, -1, -1), tc], 1).contiguous()
    state = torch.full((B, N + 1), V, dtype=torch.int64, device=DEV)
    state[:, 1:P + 1] = ctx_codes.to(DEV)
    out_c = torch.zeros(B, N, dtype=torch.int64, device=DEV)
    out_l = torch.zeros(B, N, V, device=DEV)
    lib = L.lib()
    pl = plm._plan_get(tc.device, N)
    m = C.byref(pl.struct)
    ws = ops.workspace(lib.mtts_plm_infer_workspace_bytes(m, B, N), tc.device)
    L.check(lib.mtts_plm_infer_range_f32(m, cat.data_ptr(), cat.stride(0), cat.stride(1), B, N, P, N, state.data_ptr(),
                                         out_c.data_ptr(), out_l.data_ptr(), ws.data_ptr(), ws.numel(), ops._stream()))
    assert torch.equal(out_c[:, P:], codes) and torch.equal(out_l[:, P:], logits)


def test_empty_context_is_infer(tts):
    plm = tts.plm
    tc = torch.randn(3, 11, 512, generator=gen(5)).abs().to(DEV)
    empty = PLMContext(torch.zeros(1, 0, 512, device=DEV), torch.zeros(1, 0, dtype=torch.int64, device=DEV))
    with graphs.disabled():
        ref = plm.infer(tc, return_logits=True)
        got = plm.infer(tc, return_logits=True, context=empty)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])


@pytest.mark.parametrize("causal", [False, True])
def test_shared_context_equals_repeated_rows(tts, causal):
    plm = tts.plm
    ctx_tc, ctx_codes, tc = case_inputs(33, 3, 1)
    dec = plm.infer_causal if causal else plm.infer
    with graphs.disabled():
        one = dec(tc[:, :12].to(DEV), return_logits=True, context=context(ctx_tc, ctx_codes))
        rep = dec(tc[:, :12].to(DEV), return_logits=True, context=context(ctx_tc.repeat(3, 1, 1), ctx_codes.repeat(3, 1)))
    assert torch.equal(one[0], rep[0]) and torch.equal(one[1], rep[1])


SAMPLINGS = [None, Sampling(temperature=0.9, top_k=40, seed=5)]


@pytest.mark.parametrize("smp", range(len(SAMPLINGS)))
def test_ranges_equal_the_whole_decode(tts, smp):
    plm, sampling = tts.plm, SAMPLINGS[smp]
    ctx_tc, ctx_codes, tc = case_inputs(20, 3, 3)
    T = 13
    tc = tc[:, :T].to(DEV)
    ctx = context(ctx_tc, ctx_codes)
    kw = {} if sampling is None else dict(sampling=sampling, keys=torch.arange(4, 7))
    with graphs.disabled():
        ref_codes, ref_logits = plm.infer(tc, return_logits=True, context=ctx, **kw)
    rng = random.Random(smp)
    for graphed in (False, True):
        for cuts in ([0, T], list(range(T + 1)), [0] + sorted(rng.sample(range(1, T), 3)) + [T]):
            for rep in range(3 if graphed else 1):
                dec = plm.begin_decode(tc, context=ctx, **kw)
                codes, logits = [], []
                for t1 in cuts[1:]:
                    if graphed:
                        c, lg = plm.decode_until(dec, t1, return_logits=True)
                    else:
                        with graphs.disabled():
                            c, lg = plm.decode_until(dec, t1, return_logits=True)
                    codes.append(c)
                    logits.append(lg)
                assert torch.equal(torch.cat(codes, 1), ref_codes), (graphed, cuts, rep)
                assert torch.equal(torch.cat(logits, 1), ref_logits), (graphed, cuts, rep)
                assert torch.equal(dec.codes, ref_codes) and torch.equal(dec.target, ref_codes)


def test_replay_with_a_new_context_needs_no_capture(tts):
    plm = tts.plm
    ctx_tc, ctx_codes, tc = case_inputs(16, 4, 1)
    tc = tc[:, :10].to(DEV)
    for _ in range(2):                                                      # warm-up, capture
        plm.infer(tc, context=context(ctx_tc, ctx_codes))
    n_graphs, n_replayed = len(plm._graphs().cache), graphs.replayed_launches
    outs = set()
    for s in range(4):
        c2_tc, c2_codes, _ = case_inputs(16, 4, 1)
        c2_tc = c2_tc * (1 + s)
        c2_codes = (c2_codes + 97 * s) % CFG["vq_bins"]
        got = plm.infer(tc, context=context(c2_tc, c2_codes))
        with graphs.disabled():
            want = plm.infer(tc, context=context(c2_tc, c2_codes))
        assert torch.equal(got, want), s
        outs.add(tuple(got.flatten().tolist()))
    assert len(plm._graphs().cache) == n_graphs and graphs.replayed_launches > n_replayed
    assert len(outs) > 1                                                    # the context did change the codes


# ------------------------------------------------------------------------------ causal prefill
@pytest.mark.parametrize("engine", ["f16x2", "bf16x3"])
@pytest.mark.parametrize("P,B", [(7, 3), (64, 1), (130, 3)])
def test_prefill_agrees_with_single_row_steps(tts, engine, P, B):
    """The plain causal decode of cat(ctx_tc, tc) fills its caches one row per step; taking its first P codes as the context
    codes makes it the context decode with a P-step prefill.  The once-through prefill gives the same codes (up to
    near-ties) and logits within 2e-3."""
    plm, T = tts.plm, 12
    ctx_tc, _, tc = case_inputs(P, B, B)
    cat = torch.cat([ctx_tc, tc[:, :T]], 1).to(DEV)
    with pack.engine_scope(ENGINES[engine]):
        steps_codes, steps_logits = plm.infer_causal(cat, return_logits=True)
        ctx = PLMContext(ctx_tc.to(DEV), steps_codes[:, :P].contiguous())
        codes, logits = plm.infer_causal(tc[:, :T].to(DEV), return_logits=True, context=ctx)
    err = (logits - steps_logits[:, P:]).abs().max().item()
    assert err <= TOL, err
    for b in range(B):
        for j in range(T):
            if int(codes[b, j]) != int(steps_codes[b, P + j]):
                assert near_tie(steps_logits[b, P + j].cpu()), (b, j)
                break
    helpers.record("plm_context_prefill", dict(engine=engine, P=P, B=B, max_abs=err))


# ------------------------------------------------------------------------------ sampling
@pytest.mark.parametrize("causal", [False, True])
def test_sampled_picks(tts, causal):
    """Picks equal the sampler's oracle on the device's own logits at target step j, and the device sampler's draw at step j
    (what infer's step j draws); temperature 0 gives the greedy ids."""
    plm = tts.plm
    ctx_tc, ctx_codes, tc = case_inputs(40, 3, 1)
    tc = tc[:, :16].to(DEV)
    ctx = context(ctx_tc, ctx_codes)
    dec = plm.infer_causal if causal else plm.infer
    s = Sampling(temperature=1.1, top_k=60, top_p=0.95, seed=2 ** 63 + 9)
    keys = torch.tensor([3, 2 ** 40, 7])
    codes, logits = dec(tc, return_logits=True, sampling=s, keys=keys, context=ctx)
    for j in range(tc.shape[1]):
        assert torch.equal(ops.sample_rows(logits[:, j].contiguous(), j, s, keys), codes[:, j]), j
        want, gaps = RS.sample_rows(logits[:, j].cpu().numpy(), j, s.temperature, s.top_k, s.top_p, s.seed, keys.numpy())
        for b in range(3):
            assert int(codes[b, j]) == int(want[b]) or gaps[b] <= NEAR, (j, b)
    greedy = dec(tc, context=ctx)
    assert torch.equal(dec(tc, sampling=Sampling(temperature=0.0, seed=4), context=ctx), greedy)


# ------------------------------------------------------------------------------ through the pipeline
def _e2e_inputs(durations):
    phone = torch.randint(0, 320, (3, 9), generator=gen(61)).to(DEV)
    melp = (torch.randn(3, 56, 80, generator=gen(62)) * 2 - 4).to(DEV)
    forced = (torch.full((3, 9), 4, dtype=torch.int32) if durations == "equal" else
              torch.randint(1, 7, (3, 9), generator=gen(65), dtype=torch.int32)).to(DEV)
    return phone, melp, forced


def _prompt_context(tts, seed, Bc=1):
    phone = torch.randint(0, 320, (Bc, 7), generator=gen(seed)).to(DEV)
    d = torch.randint(1, 12, (1, 7), generator=gen(seed + 1), dtype=torch.int32).repeat(Bc, 1).to(DEV)
    mel_prompt = (torch.randn(Bc, int(d[0].sum()) + 5, 80, generator=gen(seed + 2)) * 2 - 4).to(DEV)
    mel_timbre = (torch.randn(Bc, 48, 80, generator=gen(seed + 3)) * 2 - 4).to(DEV)
    return tts.generator.plm_context(phone, d, mel_prompt, mel_timbre), (phone, d, mel_prompt, mel_timbre)


def test_plm_context_is_the_datasets_read_latent(tts):
    """MegaG.plm_context equals s2_latent followed by the dataset's expand-and-pool (datamodule.py:163-178), restated."""
    ctx, (phone, d, mel_prompt, mel_timbre) = _prompt_context(tts, 80, Bc=2)
    n = int(d[0].sum())
    lens = torch.full((2,), phone.shape[1], dtype=torch.int32, device=DEV)
    with torch.no_grad():
        tc, codes = tts.generator.s2_latent(phone, lens, mel_timbre, mel_prompt[:, :n])
    tce = R.length_regulate(tc.cpu(), d.cpu())
    tc8 = torch.nn.functional.max_pool1d(tce.transpose(1, 2), 8, ceil_mode=True).transpose(1, 2)
    assert ctx.P == -(-n // 8) and tuple(codes.shape) == (1, 2, ctx.P)
    assert torch.equal(ctx.tc8.cpu(), tc8) and torch.equal(ctx.codes, codes[0])
    with pytest.raises(L.MttsError):                                          # unequal sum(d)
        tts.generator.plm_context(phone, torch.cat([d[:1], d[1:] + 1]), mel_prompt, mel_timbre)
    with pytest.raises(L.MttsError):                                          # a mel shorter than sum(d)
        tts.generator.plm_context(phone, d, mel_prompt[:, :n - 1], mel_timbre)


@pytest.mark.parametrize("causal", [False, True])
def test_synthesize_decodes_with_the_context(tts, causal):
    phone, melp, forced = _e2e_inputs("equal")
    ctx, _ = _prompt_context(tts, 90)
    smp = dict(sampling=Sampling(temperature=0.9, top_k=50, seed=17), keys=torch.arange(3))
    out = tts.synthesize(phone, melp, forced_durations=forced, plm_context=[ctx, ctx], causal_decode=causal,
                         return_intermediates=True, **smp)
    plain = tts.synthesize(phone, melp, forced_durations=forced, causal_decode=causal, return_intermediates=True, **smp)
    dec = tts.plm.infer_causal if causal else tts.plm.infer
    with torch.no_grad():
        codes = dec(out["tc8"], context=[ctx, ctx], **smp)
        mel = tts.generator.decode_mel_cl(out["tc_latent_expand"], codes)
    assert torch.equal(out["p_codes"], codes) and torch.equal(out["mel"], mel)
    assert torch.equal(out["dt"], plain["dt"]) and torch.equal(out["tc8"], plain["tc8"])
    assert not torch.equal(out["p_codes"], plain["p_codes"])
    assert out["wav"].shape == plain["wav"].shape


def _run_stream(tts, *args, **kw):
    chunks = list(tts.synthesize_stream(*args, **kw))
    assert chunks[-1]["last"]
    return chunks, torch.cat([c["wav"] for c in chunks], -1)


@pytest.mark.parametrize("durations", ["equal", "ragged"])
@pytest.mark.parametrize("prompt", [False, True])
def test_stream_equals_synthesize(tts, durations, prompt):
    phone, melp, forced = _e2e_inputs(durations)
    ctx, _ = _prompt_context(tts, 100)
    kw = dict(forced_durations=forced, prompt_mels=melp if prompt else None, plm_context=ctx,
              sampling=Sampling(temperature=0.9, top_k=50, seed=17), keys=torch.arange(3, 6))
    ref = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    if durations == "ragged":
        assert len(set(ref["totals"])) > 1
    for cf in (8, max(ref["totals"]) + 100):
        chunks, wav = _run_stream(tts, phone, melp, chunk_frames=cf, **kw)
        assert torch.equal(chunks[-1]["p_codes"], ref["p_codes"])
        assert wav.shape == ref["wav"].shape
        err = (wav - ref["wav"]).abs().max().item()
        assert err <= 1e-5, (cf, err)


def test_rejected_combinations(tts):
    phone, melp, forced = _e2e_inputs("equal")
    ctx, _ = _prompt_context(tts, 110)
    pros = [(torch.randn(3, 40, 80, generator=gen(63)) * 2 - 3).to(DEV)]
    with pytest.raises(L.MttsError):
        tts.synthesize(phone, melp, forced_durations=forced, plm_context=ctx, prosody_mels=pros, prosody_weights=[1, 1])
    with pytest.raises(L.MttsError):
        tts.synthesize_stream(phone, melp, plm_context=ctx, prosody_mels=pros, prosody_weights=[1, 1])
    with pytest.raises(L.MttsError):
        tts.synthesize_many([(phone[0], melp[0])], plm_context=ctx)
    two = PLMContext(ctx.tc8.repeat(2, 1, 1), ctx.codes.repeat(2, 1))                  # Bc = 2 for B = 3
    with pytest.raises(L.MttsError):
        tts.synthesize(phone, melp, forced_durations=forced, plm_context=two)
    big = PLMContext(ctx.tc8, torch.full_like(ctx.codes, CFG["vq_bins"]))            # a code outside [0, vq_bins)
    with pytest.raises(L.MttsError):
        tts.plm.infer(torch.zeros(3, 4, 512, device=DEV), context=big)
    with pytest.raises(L.MttsError):
        tts.plm.infer(torch.zeros(3, 4, 512, device=DEV), context=PLMContext(torch.zeros(1, 2, 256, device=DEV),
                                                                             torch.zeros(1, 2, dtype=torch.int64,
                                                                                         device=DEV)))
