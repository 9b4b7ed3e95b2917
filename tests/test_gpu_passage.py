"""GPU: long-form synthesis.  The ragged row copy (csrc/ops.cu, copy_row_segments_kernel) against torch slicing,
MRTE.tc_latent with a cached prompt encoding, and Megatts.synthesize_passage / synthesize_passage_stream against
synthesize, MegaPLM.infer with hand-built context windows, and the vocoder over hand-assembled passage mels.

Every check is bit for bit, except the stream's chunks against the whole call (1e-5: a vocoder window can take another
tensor-core plan than the whole passage)."""
import pytest
import torch

import helpers
import ref_passage as RP
from megatts2_b200 import graphs, ops, pack
from megatts2_b200 import passage as PS
from megatts2_b200.models.megatts2 import PLMContext
from megatts2_b200.sampling import Sampling

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]
DEV = "cuda"
ENGINES = pytest.mark.parametrize("engine", [pack.ENGINE_F16X2, pack.ENGINE_BF16X3, pack.ENGINE_FFMA],
                                  ids=["f16x2", "bf16x3", "ffma"])
HOP, PAD = 256, 5


def gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def tts(weights_cpu):
    return helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)


# ------------------------------------------------------------------------------ kernel
def _copy_ref(dst, src, src_off, dst_off, n, fill=None):
    out = dst.clone()
    for b in range(dst.shape[0]):
        for r in range(max(n[b], 0)):
            d, s = dst_off[b] + r, (src_off[b] + r if src is not None else 0)
            if not 0 <= d < dst.shape[1] or (src is not None and not 0 <= s < src.shape[1]):
                continue
            if src is None:
                out[b, d] = fill
            else:
                out[b, d] = src[b if src.shape[0] > 1 else 0, s]
    return out


@pytest.mark.parametrize("row_bytes", [4, 8, 12, 320, 2048])
@pytest.mark.parametrize("B", [1, 5, 64])
@pytest.mark.parametrize("aligned", [True, False])
def test_copy_row_segments_against_slicing(row_bytes, B, aligned):
    """Random tables with unaligned offsets, n = 0 and entries running past either buffer or below row 0.  dst is a
    window of an over-allocated buffer whose canary rows (and, unaligned, a canary word per row) must not change."""
    g = gen(row_bytes + B)
    w, rows_s, rows_d, c = row_bytes // 4, 23, 31, 4
    extra = 0 if aligned else 1
    big = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, rows_d + 2 * c, w + extra), generator=g, dtype=torch.int32).to(DEV)
    src_big = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, rows_s, w + extra), generator=g, dtype=torch.int32).to(DEV)
    dst, src = big[:, c:c + rows_d, extra:], src_big[:, :, extra:]
    n = torch.randint(0, 20, (B,), generator=g).tolist()
    n[0] = 0
    s_off = torch.randint(-3, rows_s, (B,), generator=g).tolist()
    d_off = torch.randint(-3, rows_d, (B,), generator=g).tolist()
    for bsrc in (src, src[:1]):
        before = big.clone()
        want = _copy_ref(dst, bsrc, s_off, d_off, n)
        ops.copy_row_segments(dst, d_off, n, src=bsrc, src_off=s_off)
        assert torch.equal(dst, want)
        mask = torch.ones_like(big, dtype=torch.bool)
        mask[:, c:c + rows_d, extra:] = False
        assert torch.equal(big[mask], before[mask])                      # canaries
        big.copy_(before)
    f32 = dst.view(torch.float32)
    want = _copy_ref(f32, None, None, d_off, n, fill=PS.SILENCE)
    ops.copy_row_segments(f32, d_off, n, fill=PS.SILENCE)
    assert torch.equal(dst, want.view(torch.int32))                      # compared as bits: random words hold NaNs


def test_copy_row_segments_int64_codes():
    codes = torch.arange(64 * 9, dtype=torch.int64, device=DEV).reshape(64, 9)
    dst = torch.full((64, 12), -7, dtype=torch.int64, device=DEV)
    off = [b % 5 for b in range(64)]
    n = [b % 9 for b in range(64)]
    want = _copy_ref(dst, codes, off, [1] * 64, n)
    ops.copy_row_segments(dst, [1] * 64, n, src=codes, src_off=off)
    assert torch.equal(dst, want)


# ------------------------------------------------------------------------------ MRTE with a cached prompt encoding
@ENGINES
def test_tc_latent_with_mel_context(tts, engine):
    phone = torch.randint(0, 320, (3, 11), generator=gen(1)).to(DEV)
    mel = (torch.randn(3, 56, 80, generator=gen(2)) * 2 - 4).to(DEV)
    mrte = tts.generator.mrte
    with pack.engine_scope(engine), torch.no_grad():
        want = mrte.tc_latent(phone, mel)
        enc = mrte.encode_prompt(mel)
        assert torch.equal(mrte.tc_latent(phone, mel_context=enc), want)
        assert torch.equal(mrte.tc_latent(phone, mel, mel_context=enc), want)


# ------------------------------------------------------------------------------ passages
B = 3


def _passage(Tps=(7, 9, 5), seed=10):
    sents = [torch.randint(0, 320, (B, t), generator=gen(seed + i)).to(DEV) for i, t in enumerate(Tps)]
    melp = (torch.randn(B, 56, 80, generator=gen(seed + 50)) * 2 - 4).to(DEV)
    return sents, melp


def _ctx(Bc, P=6, seed=70):
    return PLMContext(torch.rand(Bc, P, 512, generator=gen(seed)).to(DEV),
                      torch.randint(0, 1024, (Bc, P), generator=gen(seed + 1)).to(DEV))


SMP = Sampling(temperature=0.9, top_k=50, seed=17)


@ENGINES
@pytest.mark.parametrize("sampled", [False, True])
def test_one_sentence_passage_is_synthesize(tts, engine, sampled):
    sents, melp = _passage((9,))
    kw = dict(sampling=SMP, keys=torch.tensor([5, -3, 2 ** 40])) if sampled else {}
    with pack.engine_scope(engine):
        ref = tts.synthesize(sents[0], melp, return_intermediates=True, **kw)
        out = tts.synthesize_passage(sents, melp, return_intermediates=True, **kw)
    s = out["sentences"][0]
    assert torch.equal(s["dt"], ref["dt"]) and torch.equal(s["p_codes"], ref["p_codes"])
    assert torch.equal(out["mel"], ref["mel"]) and torch.equal(out["wav"], ref["wav"])
    assert out["wav_lens"] == ref["wav_lens"] and out["context_rows_used"].tolist() == [0]


@ENGINES
def test_independent_sentences(tts, engine):
    sents, melp = _passage()
    with pack.engine_scope(engine):
        out = tts.synthesize_passage(sents, melp, context_rows=0, pause_frames=3, return_intermediates=True)
        for i, ph in enumerate(sents):
            ref = tts.synthesize(ph, melp, return_intermediates=True)
            s = out["sentences"][i]
            assert torch.equal(s["dt"], ref["dt"]) and torch.equal(s["p_codes"], ref["p_codes"]), i
            for b in range(B):
                f, L = int(out["frame_offsets"][b, i]), ref["totals"][b]
                assert torch.equal(out["mel"][b, f:f + L], ref["mel"][b, :L]), (i, b)
    assert out["context_rows_used"].tolist() == [0, 0, 0]


def _hand_window(initial, sents_out, context_rows):
    """The window of the next sentence, built with torch slicing from the earlier sentences' outputs (ref_passage)."""
    P0 = 0 if initial is None else initial.P
    P, rows = RP.window(P0, [s["totals"] for s in sents_out], context_rows)
    if not sents_out:
        if P == 0:
            return None, 0
        return PLMContext(initial.tc8[:, P0 - P:].expand(B, -1, -1).contiguous(),
                          initial.codes[:, P0 - P:].expand(B, -1).contiguous()), P
    if P == 0:
        return None, 0
    tc8, codes = [], []
    for b, row in enumerate(rows):
        t, c = [], []
        for src, j in row:
            if src == "ctx":
                bb = b if initial.tc8.shape[0] > 1 else 0
                t.append(initial.tc8[bb, j])
                c.append(initial.codes[bb, j])
            else:
                t.append(sents_out[src]["tc8"][b, j])
                c.append(sents_out[src]["p_codes"][b, j])
        tc8.append(torch.stack(t))
        codes.append(torch.stack(c))
    return PLMContext(torch.stack(tc8), torch.stack(codes)), P


@ENGINES
@pytest.mark.parametrize("initial", [None, 1, B])
@pytest.mark.parametrize("context_rows", [128, 5])
def test_window_matches_infer_with_hand_built_context(tts, engine, initial, context_rows):
    sents, melp = _passage()
    ctx = None if initial is None else _ctx(initial)
    with pack.engine_scope(engine):
        out = tts.synthesize_passage(sents, melp, plm_context=ctx, context_rows=context_rows, return_intermediates=True)
        assert any(len(set(s["totals"])) > 1 for s in out["sentences"])          # ragged totals
        for i, s in enumerate(out["sentences"]):
            W, P = _hand_window(ctx, out["sentences"][:i], context_rows)
            assert int(out["context_rows_used"][i]) == P
            with torch.no_grad():
                want = tts.plm.infer(s["tc8"], context=W)
            assert torch.equal(s["p_codes"], want), i


@ENGINES
def test_sampled_sentence_is_synthesize_with_shifted_keys(tts, engine):
    sents, melp = _passage()
    keys = torch.tensor([3, 2 ** 63 - 2 ** 32, -1])
    ctx = _ctx(1)
    with pack.engine_scope(engine):
        out = tts.synthesize_passage(sents, melp, plm_context=ctx, sampling=SMP, keys=keys, return_intermediates=True)
        for i, ph in enumerate(sents):
            W, _ = _hand_window(ctx, out["sentences"][:i], 128)
            ki = torch.tensor([RP.key(k, i) for k in keys.tolist()])
            ref = tts.synthesize(ph, melp, plm_context=W, sampling=SMP, keys=ki, return_intermediates=True)
            s = out["sentences"][i]
            assert torch.equal(s["dt"], ref["dt"]) and torch.equal(s["p_codes"], ref["p_codes"]), i
            for b in range(B):
                f, L = int(out["frame_offsets"][b, i]), ref["totals"][b]
                assert torch.equal(out["mel"][b, f:f + L], ref["mel"][b, :L]), (i, b)


@ENGINES
def test_waveform_is_the_vocoder_over_the_assembled_mel(tts, engine):
    sents, melp = _passage()
    pauses = [[0, 7], [12, 1], [3, 30]]
    with pack.engine_scope(engine):
        out = tts.synthesize_passage(sents, melp, pause_frames=pauses, return_intermediates=True)
        totals = [s["totals"] for s in out["sentences"]]
        frames, offsets = RP.layout(totals, pauses)
        assert out["frame_offsets"].tolist() == offsets
        F = [len(f) for f in frames]
        assert out["wav_lens"] == [HOP * (f + 2 * PAD) for f in F]
        for b in range(B):
            mel = torch.empty(F[b], 80, device=DEV)
            for k, e in enumerate(frames[b]):
                mel[k] = PS.SILENCE if e[0] == "pause" else out["mel"][b, offsets[b][e[1]] + e[2]]
            assert torch.equal(out["mel"][b, :F[b]], mel), b
            with torch.no_grad():
                w = tts.hifi_gan.decode_batch_cl(mel[None])
            assert torch.equal(out["wav"][b, :, :w.shape[-1]], w[0]), b
            assert not out["wav"][b, :, w.shape[-1]:].any()


@pytest.mark.parametrize("pause", [0, 40])
@pytest.mark.parametrize("engine", [pack.ENGINE_F16X2, pack.ENGINE_BF16X3], ids=["f16x2", "bf16x3"])
def test_stream_equals_whole_call(tts, pause, engine):
    sents, melp = _passage()
    kw = dict(pause_frames=pause, sampling=SMP, plm_context=_ctx(B))
    with pack.engine_scope(engine):
        ref = tts.synthesize_passage(sents, melp, return_intermediates=True, **kw)
        chunks = list(tts.synthesize_passage_stream(sents, melp, **kw))
    assert [c["sentence"] for c in chunks] == list(range(len(sents))) and chunks[-1]["last"]
    last = chunks[-1]
    assert last["wav_lens"] == ref["wav_lens"] and torch.equal(last["mel"], ref["mel"])
    assert torch.equal(last["frame_offsets"], ref["frame_offsets"])
    for b in range(B):
        pos = 0
        row = []
        for c in chunks:
            assert c["offset"][b] == pos
            row.append(c["wav"][b, 0, :c["valid"][b]])
            assert not c["wav"][b, 0, c["valid"][b]:].any()
            pos += c["valid"][b]
        assert pos == ref["wav_lens"][b]
        err = (torch.cat(row) - ref["wav"][b, 0, :pos]).abs().max().item()
        assert err <= 1e-5, (b, err)


def test_stream_yields_each_chunk_after_its_sentence_when_pauses_cover_the_halo(tts, monkeypatch):
    """With pauses of at least the vocoder's halo, chunk i comes before sentence i + 1 runs; with shorter ones, after."""
    sents, melp = _passage()
    hv = tts.hifi_gan.generator.receptive_field()
    for pause, lag in ((hv, 0), (hv - 1, 1)):
        log = []
        real = PS.run_sentences

        def logged(*a, **k):
            for i, x in enumerate(real(*a, **k)):
                log.append(("sentence", i))
                yield x
        monkeypatch.setattr(PS, "run_sentences", logged)
        for c in tts.synthesize_passage_stream(sents, melp, pause_frames=pause):
            log.append(("chunk", c["sentence"]))
        monkeypatch.setattr(PS, "run_sentences", real)
        for i in range(len(sents) - 1):
            assert log.index(("chunk", i)) > log.index(("sentence", min(i + lag, len(sents) - 1))), (pause, log)
            if i + lag + 1 < len(sents):
                assert log.index(("chunk", i)) < log.index(("sentence", i + lag + 1)), (pause, log)


def test_passage_leaves_graph_caches_alone(tts):
    sents, melp = _passage()
    with torch.no_grad():
        tts.synthesize(sents[0], melp)
        tts.synthesize(sents[0], melp)
    before = {m: {k: dict(v.cache) for k, v in getattr(getattr(tts, m), "_graph_caches", {}).items()}
              for m in ("plm", "adm")}
    tts.synthesize_passage(sents, melp)
    list(tts.synthesize_passage_stream(sents, melp))
    after = {m: {k: dict(v.cache) for k, v in getattr(getattr(tts, m), "_graph_caches", {}).items()}
             for m in ("plm", "adm")}
    assert before.keys() == after.keys()
    for m in before:
        assert before[m].keys() == after[m].keys()
        for k in before[m]:
            assert list(before[m][k]) == list(after[m][k])
            assert all(before[m][k][kk] is after[m][k][kk] for kk in before[m][k])
    assert graphs.enabled()


def test_range_flag_redoes_each_sentence_on_bf16x3(golden, weights_cpu):
    """test_synthesize_attention_overflow_reruns_finite_on_bf16x3's overflow (the first PLM layer's queries x 2^17, keys
    x 2^-17) in a 3-sentence passage under f16x2: the passage warns and redoes every sentence on bf16x3, and equals the
    same model's passage with the sentences under bf16x3 and the vocoder on f16x2 (its .engine set by hand).  Its first
    sentence, which has no context, also equals the unscaled model's."""
    g = golden("e2e")
    melp = g["mel_prompt"].to(DEV)
    sents = [torch.randint(0, 320, (1, t), generator=gen(13 + t)).to(DEV) for t in (70, 66, 72)]
    forced = [torch.full((1, s.shape[1]), 8, dtype=torch.int32, device=DEV) for s in sents]
    scaled = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    lyr = scaled.plm.plm.layers[0]
    with torch.no_grad():
        lyr.attn.w_q.weight.mul_(2.0 ** 17)
        lyr.attn.w_k.weight.mul_(2.0 ** -17)
    ops.tc_overflow(torch.device(DEV))
    with pack.engine_scope(pack.ENGINE_F16X2):
        with pytest.warns(UserWarning, match="fp16 range") as rec:
            got = scaled.synthesize_passage(sents, melp, forced_durations=forced, pause_frames=4,
                                            return_intermediates=True)
    assert sum("sentence" in str(w.message) for w in rec) == 3
    plain = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    with pack.engine_scope(pack.ENGINE_BF16X3):
        first = plain.synthesize(sents[0], melp, forced_durations=forced[0], return_intermediates=True)
    assert torch.equal(got["sentences"][0]["p_codes"], first["p_codes"])
    scaled.hifi_gan.generator.engine = pack.ENGINE_F16X2
    with pack.engine_scope(pack.ENGINE_BF16X3):
        want = scaled.synthesize_passage(sents, melp, forced_durations=forced, pause_frames=4, return_intermediates=True)
    for i in range(3):
        assert torch.equal(got["sentences"][i]["p_codes"], want["sentences"][i]["p_codes"]), i
    assert torch.equal(got["mel"], want["mel"]) and torch.equal(got["wav"], want["wav"])
    assert torch.isfinite(got["wav"]).all()
