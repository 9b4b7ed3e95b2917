"""GPU parity: the CUDA path (through the C ABI) against (1) the golden fixtures written by the
REAL reference, (2) the CPU oracle on seeded inputs, (3) size-independent properties.

Bars: integer outputs (VQ codes, PLM ids, durations, gather indices) bit-exact; floating
point within the tolerance written next to each check (fp32 vs fp32 with different
summation order; the noise floors are in SURVEY.md §7.2)."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers
from oracle import ref_megatts2 as R
from oracle import weights

pytestmark = pytest.mark.gpu
DEV = "cuda"


def gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


def maxerr(a, b):
    return (a.detach().float().cpu() - b.detach().float().cpu()).abs().max().item()


@pytest.fixture(scope="module")
def G(weights_cpu):
    return helpers.build_g(weights_cpu("g"), DEV)


@pytest.fixture(scope="module")
def PLM(weights_cpu):
    return helpers.build_plm(weights_cpu("plm"), DEV)


@pytest.fixture(scope="module")
def ADM(weights_cpu):
    return helpers.build_adm(weights_cpu("adm"), DEV)


@pytest.fixture(scope="module")
def HIFI(weights_cpu):
    return helpers.build_hifigan(weights_cpu("hifigan"), DEV)


# ------------------------------------------------------------------------------ tap-GEMM
def test_conv_linearity_property_full_size():
    """size-independent property at a BASELINE-size GEMM: f(a x1 + x2) == a f(x1) + f(x2) (no bias)."""
    from megatts2_b200 import ops
    g = torch.Generator(device=DEV)
    g.manual_seed(3)
    x1 = torch.randn(1, 4096, 1024, device=DEV, generator=g)
    x2 = torch.randn(1, 4096, 1024, device=DEV, generator=g)
    w = torch.randn(1, 1024, 4096, device=DEV, generator=g) / 32
    lhs = ops.conv1d(2.0 * x1 + x2, w, None, k=1)
    rhs = 2.0 * ops.conv1d(x1, w, None, k=1) + ops.conv1d(x2, w, None, k=1)
    assert (lhs - rhs).abs().max().item() < 5e-5
    # and against cuBLAS-free fp64 on a row sample
    rows = torch.tensor([0, 1, 777, 4095], device=DEV)
    ref = (x1[0, rows].double() @ w[0].double())
    assert (ops.conv1d(x1, w, None, k=1)[0, rows].double() - ref).abs().max().item() < 5e-5


# ------------------------------------------------------------------------------ LN
@pytest.mark.parametrize("C_", [384, 512, 768, 1024, 100])
def test_layernorm(C_):
    from megatts2_b200 import ops
    g = gen(C_)
    x = torch.randn(37, C_, generator=g) * 3 + 1
    ga, be = torch.randn(C_, generator=g), torch.randn(C_, generator=g)
    res, y0 = torch.randn(37, C_, generator=g), torch.randn(37, C_, generator=g)
    ref = F.layer_norm(x.double(), (C_,), ga.double(), be.double(), 1e-5)
    y = ops.layernorm(x.to(DEV), ga.to(DEV), be.to(DEV))
    assert maxerr(y, ref) < 1e-5
    ref2 = F.relu(ref) + res.double() + y0.double()
    y2 = ops.layernorm(x.to(DEV), ga.to(DEV), be.to(DEV), res=res.to(DEV), out=y0.clone().to(DEV), post_act=1,
                       accumulate=True)
    assert maxerr(y2, ref2) < 1e-5
    xi = x.clone().to(DEV)                  # in place
    ops.layernorm(xi, ga.to(DEV), be.to(DEV), out=xi)
    assert maxerr(xi, ref) < 1e-5


# ------------------------------------------------------------------------------ VQ
def test_vq_search_golden(golden, weights_cpu):
    from megatts2_b200 import ops
    g = golden("vq_search")
    embed = weights_cpu("g")["vqpe.vq.vq.layers.0._codebook.embed"].to(DEV)
    idx = ops.vq_argmin(g["x"].to(DEV), embed).cpu()
    ref = g["idx"]
    mism = (idx != ref)
    # a mismatch is only tolerated where fp64 itself says the two best codes are closer than fp32
    # rounding of |x|^2 + |e|^2 ~ 500 (2 ulp ~ 6e-5); everywhere else the index must be bit-exact
    assert bool((g["gap64"][mism] < 2e-4).all()), f"{int(mism.sum())} mismatches, gaps {g['gap64'][mism]}"
    rate = 1.0 - mism.float().mean().item()
    print(f"VQ-index bit-exact rate vs reference (adversarial fixture): {rate:.6f}")
    helpers.record("vq_adversarial_fixture", dict(rows=int(idx.numel()), mismatches=int(mism.sum()), bit_exact_rate=rate,
                                                  max_gap64_of_a_mismatch=float(g["gap64"][mism].max()) if mism.any() else 0.0))
    # the fixture's second block is BUILT from near-ties (fp64 gap of the two best codes below fp32 rounding of
    # |x|^2 + |e|^2 ~ 500); measured on H100: 0 mismatches of 1088 rows, so the bar is 1.0
    assert rate == 1.0
    assert torch.equal(idx[:512], ref[:512])                 # the random (non-adversarial) block
    assert torch.equal(idx[-64:], torch.arange(64))          # exact codes map to themselves
    dec = ops.vq_gather(ref.view(1, -1).to(DEV), embed)
    assert torch.equal(dec.cpu()[0], embed.cpu()[ref])
    rep = ops.vq_gather(ref[:10].view(2, 5).to(DEV), embed, t_out=37, repeat=8)
    ref_rep = embed.cpu()[ref[:10].view(2, 5)].repeat_interleave(8, dim=1)[:, :37]
    assert torch.equal(rep.cpu(), ref_rep)


def test_vq_full_size_property(weights_cpu):
    """C4-size search (64 x 64 rows): result must be the exact fp64 nearest code wherever the gap is clear,
    and quantising a code row must return that code (idempotence)."""
    from megatts2_b200 import ops
    embed = weights_cpu("g")["vqpe.vq.vq.layers.0._codebook.embed"]
    x = torch.randn(4096, 256, generator=gen(5))
    idx = ops.vq_argmin(x.to(DEV), embed.to(DEV)).cpu()
    d = torch.cdist(x.double(), embed.double()).pow(2)
    top2 = d.topk(2, largest=False)
    clear = (top2.values[:, 1] - top2.values[:, 0]) > 2e-4
    assert torch.equal(idx[clear], top2.indices[clear, 0])
    assert clear.float().mean() > 0.99
    again = ops.vq_argmin(embed.to(DEV)[idx.to(DEV)], embed.to(DEV)).cpu()
    assert torch.equal(again, idx)


# ------------------------------------------------------------------------------ mel front end
def test_mel_golden_and_oracle(golden):
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    g = golden("mel_frontend")
    out = extract_mel_spec(g["wav"].to(DEV))
    assert out.shape == (3, 80, 16)
    assert maxerr(out, g["mel"]) < 5e-5                      # log-mel, fp32 FFT vs pocketfft fp32
    assert (out.cpu() - g["mel"]).abs().mean().item() < 1e-5
    wav = torch.rand(5, 48000, generator=gen(21)) * 2 - 1    # C2 shape: 3-s clips
    ref = R.mel_spectrogram(wav)
    out = extract_mel_spec(wav.to(DEV))
    assert out.shape == (5, 80, 188)
    assert (out.cpu() - ref).abs().mean().item() < 1e-5      # north-star: mel L1 <= 1e-4
    assert maxerr(out, ref) < 1e-4
    fm = extract_mel_spec(wav.to(DEV), frames_major=True)
    assert torch.equal(fm.transpose(1, 2), out)
    one = extract_mel_spec(wav[0].to(DEV))
    assert torch.equal(one, out[0])
    odd = torch.rand(2, 5000, generator=gen(22)) - 0.5       # frame count not a multiple of the CTA tile
    assert maxerr(extract_mel_spec(odd.to(DEV)), R.mel_spectrogram(odd)) < 1e-4


def test_mel_linear_domain_scaling_property():
    """mel(a*x) = mel(x) + log(a) away from the clamp floor (the front end is linear before the log)."""
    from megatts2_b200.modules.tokenizer import extract_mel_spec
    wav = torch.rand(64, 48000, generator=gen(23), device="cpu").to(DEV) * 2 - 1
    a = extract_mel_spec(wav)
    b = extract_mel_spec(wav * 0.25)
    assert (b - (a + math.log(0.25))).abs().max().item() < 1e-4


# ------------------------------------------------------------------------------ small ops
def test_small_ops(golden):
    from megatts2_b200 import ops
    g = gen(31)
    x = torch.randn(2, 61, 384, generator=g)
    y = ops.maxpool_time(x.to(DEV), 8)
    assert torch.equal(y.cpu(), F.max_pool1d(x.transpose(1, 2), 8, ceil_mode=True).transpose(1, 2))
    ids = torch.randint(0, 320, (3, 17), generator=g)
    tab = torch.randn(320, 512, generator=g)
    pe = R.sine_pe_table(4000, 512)
    e = ops.embed_pe(ids.to(DEV), tab.to(DEV), pe.to(DEV), 1.0)
    assert maxerr(e, tab[ids] + pe[None, :17]) == 0.0
    assert torch.equal(ops.add_pe(x[..., :512 - 128].contiguous().to(DEV), R.sine_pe_table(100, 384).to(DEV)).cpu(),
                       x[..., :384] * 1.0 + R.sine_pe_table(100, 384)[None, :61])
    lr = golden("length_regulator")
    out, tot = ops.length_regulate(lr["x"].to(DEV), lr["d"].to(DEV))
    assert out.shape == (2, 11, 128)                          # the reference's own test (modules/mrte.py:187-194)
    assert torch.equal(out.cpu(), lr["y"]) and tot.tolist() == [10, 11]
    d = torch.randint(0, 9, (4, 33), generator=g, dtype=torch.int32)
    xx = torch.randn(4, 33, 512, generator=g)
    out, tot = ops.length_regulate(xx.to(DEV), d.to(DEV))
    assert torch.equal(out.cpu(), R.length_regulate(xx, d))
    cf = torch.randn(3, 80, 45, generator=g)
    cl = ops.to_channels_last(cf.to(DEV))
    assert torch.equal(cl.cpu(), cf.transpose(1, 2))
    assert torch.equal(ops.to_channels_first(cl).cpu(), cf)
    padded = ops.to_channels_last(cf.to(DEV), pad_rep=5)
    assert torch.equal(padded.cpu(), F.pad(cf, (5, 5), mode="replicate").transpose(1, 2))


# ------------------------------------------------------------------------------ modules vs golden
def test_encoder_golden(golden, G, PLM):
    g = golden("encoder")
    y = G.mrte.phone_encoder(g["x_phone"].to(DEV))
    assert maxerr(y, g["y_phone"]) < 1e-4
    lens = torch.tensor([7, 7], dtype=torch.int32, device=DEV)
    assert maxerr(PLM.plm(g["x_plm"].to(DEV), lens, causal=True), g["y_plm_causal"]) < 2e-4
    yn = PLM.plm(g["x_plm"].to(DEV))
    assert maxerr(yn, g["y_plm_nomask"]) < 2e-4
    from megatts2_b200.modules.transformer import run_encoder
    last = run_encoder(PLM.plm, list(PLM.plm.layers), g["x_plm"].to(DEV), last_row_only=True)
    assert last.shape == (2, 1, 1024)
    assert maxerr(last[:, 0], g["y_plm_nomask"][:, -1]) < 2e-4     # exact pruning == full computation
    # single layer + standalone MHA surfaces
    l0 = PLM.plm.layers[0]
    ref0 = R.encoder_layer(R.SD(weights.plm_state_dict(), "plm.layers.0."), g["x_plm"], 16, False)
    assert maxerr(l0(g["x_plm"].to(DEV)), ref0) < 1e-4
    ref_mha = R.mha(R.SD(weights.plm_state_dict(), "plm.layers.0.attn."), g["x_plm"], 16)
    assert maxerr(l0.attn(g["x_plm"].to(DEV)), ref_mha) < 1e-4


def test_vqpe_c1_bit_exact(golden, G):
    g = golden("vqpe")
    zq, commit, vql, codes = G.vqpe(g["mel1"].to(DEV))
    assert codes.shape == (1, 1, 16) and codes.dtype == torch.int64
    assert torch.equal(codes.cpu(), g["codes1"]), "C1: VQ code indices must be bit-exact"
    assert maxerr(zq, g["zq1"]) <= 1e-5
    assert commit.shape == (1, 1) and abs(float(vql) - float(g["vq_loss1"])) < 1e-3
    ze, _ = G.vqpe.encode_cl(g["mel1"].to(DEV))
    assert maxerr(ze.transpose(1, 2), g["ze1"]) < 2e-4
    zq2, _, _, codes2 = G.vqpe(g["mel2"].to(DEV))
    assert torch.equal(codes2.cpu(), g["codes2"]) and zq2.shape == (2, 61, 256)
    assert maxerr(zq2, g["zq2"]) <= 1e-5
    # reference-layout (B,C,T) surface of the conv stack
    cn = G.vqpe.convnet(g["mel1"][..., :20].transpose(1, 2).to(DEV))
    assert cn.shape == (1, 256, 16) and maxerr(cn, g["ze1"]) < 2e-4


def test_mrte_golden(golden, G):
    g = golden("mrte")
    tc = G.mrte.tc_latent(g["phone"].to(DEV), g["mel"].to(DEV))
    assert tc.shape == (2, 12, 512) and float(tc.min()) >= 0.0
    assert maxerr(tc, g["tc_latent"]) < 2e-4
    assert (tc.cpu() - g["tc_latent"]).abs().mean().item() < 2e-5
    ctx = G.mrte.mel_encoder.forward_cl(g["mel"].to(DEV))
    assert maxerr(ctx, g["mel_context"]) < 5e-4
    tc3 = G.mrte.tc_latent(g["phone"].to(DEV), torch.tensor([12, 12], device=DEV), g["mel"].to(DEV))
    assert torch.equal(tc3, tc)


def test_adm_golden(golden, ADM):
    g = golden("adm")
    dur, raw = ADM.infer(g["tc_latent"].to(DEV), return_raw=True)
    assert dur.shape == (2, 10, 1) and dur.dtype == torch.int32
    assert maxerr(raw, g["raw"][..., 0]) < 2e-3
    assert torch.equal(dur.cpu(), g["dur"]), "durations must match the reference exactly"
    one = ADM.infer(g["tc_latent"][1:2].to(DEV))
    assert torch.equal(one.cpu(), g["dur"][1:2])                  # batched == per-utterance
    lens = torch.tensor([10, 10], dtype=torch.int32, device=DEV)
    fwd, tgt = ADM(g["tc_latent"].to(DEV), g["dtok"].to(DEV), lens)
    assert maxerr(fwd, g["fwd"]) < 2e-3


def test_plm_golden(golden, PLM):
    g = golden("plm")
    ids, logits = PLM.infer(g["tc8"].to(DEV), return_logits=True)
    assert ids.shape == (2, 12) and ids.dtype == torch.int64
    assert torch.equal(ids.cpu(), g["ids"]), "PLM ids must be bit-exact"
    assert maxerr(logits, g["logits"]) < 2e-3
    ids1 = PLM.infer(g["tc8"][:1].to(DEV))
    assert torch.equal(ids1.cpu(), g["ids"][:1])
    pcodes = torch.cat([torch.full((2, 1), 1024), g["ids"]], 1).to(DEV)
    lens = torch.tensor([12, 12], dtype=torch.int32, device=DEV)
    f, tgt = PLM(g["tc8"].to(DEV), pcodes, lens)
    assert maxerr(f, g["fwd_logits"]) < 2e-3 and torch.equal(tgt.cpu(), g["ids"])


def test_hifigan_golden(golden, HIFI):
    g = golden("hifigan")
    wav = HIFI.decode_batch(g["mel"].to(DEV))
    assert wav.shape == (2, 1, 256 * 22)
    assert maxerr(wav, g["wav"]) < 1e-4                          # tanh output in [-1,1]
    assert (wav.cpu() - g["wav"]).abs().mean().item() < 1e-5


def test_e2e_golden(golden, weights_cpu):
    g = golden("e2e")
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    o = tts.synthesize(g["phone"].to(DEV), g["mel_prompt"].to(DEV), forced_durations=g["dt_used"].to(DEV),
                       return_intermediates=True)
    assert torch.equal(o["dt"].cpu(), g["dt"])
    assert torch.equal(o["p_codes"].cpu(), g["p_codes"])
    assert maxerr(o["tc_latent"], g["tc_latent"]) < 2e-4
    mel_cf = o["mel"].transpose(1, 2)
    assert (mel_cf.cpu() - g["mel"]).abs().mean().item() < 1e-4   # north-star: mel L1 <= 1e-4
    assert maxerr(mel_cf, g["mel"]) < 1e-3
    assert maxerr(o["wav"], g["wav_oracle"]) < 1e-3
    # free-running (ADM-predicted durations) gives the same thing when the clamp is not active
    wav = tts.synthesize(g["phone"].to(DEV), g["mel_prompt"].to(DEV))
    assert wav.shape[-1] == 256 * (int(g["dt"].sum()) + 10)


def test_e2e_vs_oracle_batched(weights_cpu):
    """B = 3 utterances with DIFFERENT total durations, fresh seeded inputs: every utterance of the batched CUDA run must
    equal the oracle's batch-1 run of that utterance - what the reference computes, one utterance at a time - on its
    valid region (ADVICE r1: the zero rows the LengthRegulator appends to shorter utterances must not leak into their
    mel / waveform; the decoder and the vocoder run per group of equal length)."""
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    phone = torch.randint(0, 320, (3, 9), generator=gen(41))
    melp = torch.randn(3, 80, 80, generator=gen(42)) * 2 - 4
    forced = torch.randint(1, 7, (3, 9), generator=gen(43), dtype=torch.int32)
    totals = forced.sum(1).tolist()
    assert len(set(totals)) > 1, "the fixture must be ragged"
    cfgs = (weights.G_CFG, weights.PLM_CFG, weights.ADM_CFG, weights.HIFIGAN_CFG)
    o = tts.synthesize(phone.to(DEV), melp.to(DEV), forced_durations=forced.to(DEV), return_intermediates=True)
    wav2, lens = tts.synthesize(phone.to(DEV), melp.to(DEV), forced_durations=forced.to(DEV), return_lengths=True)
    assert o["totals"] == totals and lens == [256 * (t + 10) for t in totals] and torch.equal(wav2, o["wav"])
    for b in range(3):
        ref = R.synthesize(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), phone[b:b + 1],
                           melp[b:b + 1], cfgs, forced_durations=forced[b:b + 1])
        t, t8 = totals[b], (totals[b] + 7) // 8
        assert torch.equal(o["dt"][b:b + 1].cpu(), ref["dt"])
        assert torch.equal(o["p_codes"][b:b + 1, :t8].cpu(), ref["p_codes"])
        assert maxerr(o["tc_latent"][b:b + 1], ref["tc_latent"]) < 2e-4
        assert (o["mel"][b:b + 1, :t].cpu() - ref["mel"].transpose(1, 2)).abs().mean().item() < 1e-4
        assert maxerr(o["wav"][b:b + 1, :, :lens[b]], ref["wav"]) < 1e-3
        assert float(o["wav"][b, :, lens[b]:].abs().max()) == 0.0 if lens[b] < o["wav"].shape[-1] else True


def test_prompt_revocode_and_synthesize_many(weights_cpu):
    """models/megatts2.py:371-373: the prompt is re-vocoded and prepended; synthesize_many buckets ragged inputs by
    (Tp, Tm) and returns per-utterance waveforms equal to the single-utterance runs."""
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    phone = torch.randint(0, 320, (2, 6), generator=gen(44)).to(DEV)
    melp = (torch.randn(2, 48, 80, generator=gen(45)) * 2 - 4).to(DEV)
    forced = torch.tensor([[2, 1, 3, 1, 2, 2], [1, 2, 2, 3, 1, 2]], dtype=torch.int32, device=DEV)
    plain = tts.synthesize(phone, melp, forced_durations=forced)
    both, lens = tts.synthesize(phone, melp, forced_durations=forced, prompt_mels=melp, return_lengths=True)
    pw = tts.hifi_gan.decode_batch_cl(melp)
    assert pw.shape[-1] == 256 * (48 + 10) and both.shape[-1] == pw.shape[-1] + plain.shape[-1]
    assert torch.equal(both[..., :pw.shape[-1]], pw) and torch.equal(both[..., pw.shape[-1]:], plain)
    assert lens == [pw.shape[-1] + 256 * (11 + 10)] * 2
    # ragged front door: three utterances in two buckets, results in input order
    p2 = torch.randint(0, 320, (4,), generator=gen(46)).to(DEV)
    m2 = (torch.randn(40, 80, generator=gen(47)) * 2 - 4).to(DEV)
    many = tts.synthesize_many([(phone[0], melp[0]), (p2, m2), (phone[1], melp[1])])
    singles = [tts.synthesize(phone[0:1], melp[0:1], return_lengths=True), tts.synthesize(p2[None], m2[None], return_lengths=True),
               tts.synthesize(phone[1:2], melp[1:2], return_lengths=True)]
    for got, (w, ln) in zip(many, singles):
        assert got.shape == (ln[0],) and torch.equal(got, w[0, 0, :ln[0]])
    # speechbrain's decode_batch(mel, mel_lens, hop_len) zeroes the samples past mel_lens * hop_len
    w = tts.hifi_gan.decode_batch(melp.transpose(1, 2), mel_lens=torch.tensor([48, 30]), hop_len=256)
    assert float(w[1, :, 30 * 256:].abs().max()) == 0.0 and float(w[1, :, :30 * 256].abs().max()) > 0
    assert torch.equal(w[0, :, :48 * 256], pw[0, :, :48 * 256]) and float(w[0, :, 48 * 256:].abs().max()) == 0.0


def test_overlapped_prompt_revocode(weights_cpu):
    """Megatts._synthesize with the prompt re-vocode on a side stream (SM budget V) beside MRTE + ADM on the remaining SMs
    (ops.launch_policy: complementary budgets, no PDL on the vocoder's stream, no CTA pairs on the AR stream): the waveform of
    the prompt is bit-identical to the sequential form, ids / durations equal, through eager, capture and replay passes; the
    policy is restored afterwards."""
    from megatts2_b200 import ops
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    B, Tp, Tm = 6, 24, 64
    phone = torch.randint(0, 320, (B, Tp), generator=gen(71)).to(DEV)
    melp = (torch.randn(B, Tm, 80, generator=gen(72)) * 2 - 4).to(DEV)
    forced = torch.randint(1, 4, (B, Tp), generator=gen(73)).to(torch.int32)
    forced[:, -1] += (forced.sum(1).max() - forced.sum(1)).to(torch.int32)          # equal totals: one vocoder group
    forced = forced.to(DEV)
    seq = tts.synthesize(phone, melp, forced_durations=forced, prompt_mels=melp, return_intermediates=True, overlap_prompt=False)
    n_p = 256 * (Tm + 10)
    keys = ("MEGATTS2_REVOCODE_SMS", "MEGATTS2_REVOCODE_FRAC", "MEGATTS2_REVOCODE_FROM")
    saved = {k: os.environ.get(k) for k in keys}
    try:
        for sms, frac, start in (("100", "1.0", "mrte"), ("116", "0.5", "adm"), ("0", "1.0", "mrte")):
            os.environ.update({keys[0]: sms, keys[1]: frac, keys[2]: start})
            for _ in range(3):      # eager, graph capture, replay
                ov = tts.synthesize(phone, melp, forced_durations=forced, prompt_mels=melp, return_intermediates=True,
                                    overlap_prompt=True)
                assert ops.launch_policy_now() == (0, 1, 1)
                assert torch.equal(ov["wav"][..., :n_p], seq["wav"][..., :n_p])
                assert torch.equal(ov["dt"], seq["dt"]) and torch.equal(ov["p_codes"], seq["p_codes"])
                assert maxerr(ov["tc_latent"], seq["tc_latent"]) < 1e-4
                assert maxerr(ov["wav"], seq["wav"]) < 1e-3
    finally:
        for k, v in saved.items():
            os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)


def test_graph_replay_matches_eager(PLM, ADM):
    """The AR drivers replayed from a CUDA graph (megatts2_b200/graphs.py: eager call, capture, replays) give the eager
    enqueue's ids / durations bit for bit, for new inputs too, and the replayed kernels are counted."""
    from megatts2_b200 import graphs, ops
    tc8 = F.relu(torch.randn(4, 12, 512, generator=gen(61))).to(DEV)
    tc8b = F.relu(torch.randn(4, 12, 512, generator=gen(62))).to(DEV)
    with graphs.disabled():
        ref_a, ref_b = PLM.infer(tc8), PLM.infer(tc8b)
        dref_a, dref_b = ADM.infer(tc8, return_raw=True), ADM.infer(tc8b, return_raw=True)
    PLM._graphs().clear(); ADM._graphs().clear()
    n0 = graphs.replayed_launches
    outs = [PLM.infer(tc8), PLM.infer(tc8), PLM.infer(tc8b), PLM.infer(tc8)]          # eager, capture + replay, replays
    assert all(torch.equal(o, r) for o, r in zip(outs, (ref_a, ref_a, ref_b, ref_a)))
    douts = [ADM.infer(tc8, return_raw=True), ADM.infer(tc8, return_raw=True), ADM.infer(tc8b, return_raw=True)]
    for (d, r), (dr, rr) in zip(douts, (dref_a, dref_a, dref_b)):
        assert torch.equal(d, dr) and torch.equal(r, rr)
    if graphs.enabled():
        assert graphs.replayed_launches > n0 and any(len(e) == 4 for e in PLM._graphs().cache.values())


def test_batch_invariance_property(weights_cpu, PLM):
    """Sharding property behind the multi-GPU split: any sub-batch gives bit-identical ids."""
    tc8 = F.relu(torch.randn(8, 16, 512, generator=gen(51))).to(DEV)
    full = PLM.infer(tc8)
    parts = torch.cat([PLM.infer(tc8[:3]), PLM.infer(tc8[3:])], 0)
    assert torch.equal(full, parts)
    assert torch.equal(full, PLM.infer(tc8))                    # deterministic


# ------------------------------------------------------------------ SURVEY.md 8f-1: opt-in causal KV-cache decode
def test_causal_decode_golden(golden, PLM, ADM):
    """Product infer_causal vs the fixture pinned on the real reference's teacher-forced causal forward."""
    g = golden("causal_decode")
    ids, logits = PLM.infer_causal(g["tc8"].to(DEV), return_logits=True)
    assert ids.dtype == torch.int64 and torch.equal(ids.cpu(), g["plm_ids"]), "causal ids must be bit-exact"
    assert maxerr(logits, g["plm_logits"]) < 2e-3
    assert torch.equal(PLM.infer_causal(g["tc8"][1:2].to(DEV)).cpu(), g["plm_ids"][1:2])     # batched == per-utterance
    # self-consistency on the device: ONE teacher-forced pass over the decode's own output reproduces every step
    pcodes = torch.cat([torch.full((2, 1), 1024, device=DEV), ids], 1)
    fwd, _ = PLM(g["tc8"].to(DEV), pcodes, torch.tensor([12, 12], dtype=torch.int32, device=DEV))
    assert maxerr(fwd, logits) < 2e-3 and torch.equal(fwd.argmax(-1), ids)
    # and it is NOT the reference's infer(): that one is non-causal
    assert not torch.equal(ids.cpu(), golden("plm")["ids"])
    dur, raw = ADM.infer_causal(g["tc_latent"].to(DEV), return_raw=True)
    assert dur.shape == (2, 10, 1) and dur.dtype == torch.int32
    assert maxerr(raw, g["adm_raw"][..., 0]) < 2e-3
    assert torch.equal(dur.cpu(), g["adm_dur"])


def test_causal_decode_vs_oracle_longer(weights_cpu, PLM, ADM):
    """Fresh seeded inputs, more steps than the fixture (the K/V cache crosses the 32-key tile of the attention kernel)."""
    tc8 = F.relu(torch.randn(3, 40, 512, generator=gen(61)))
    ref_ids, ref_lg = R.plm_infer_causal(R.SD(weights_cpu("plm")), tc8, weights.PLM_CFG, return_logits=True)
    ids, lg = PLM.infer_causal(tc8.to(DEV), return_logits=True)
    gap = ref_lg.topk(2, -1).values
    safe = (gap[..., 0] - gap[..., 1]) > 1e-3            # positions whose argmax is not a numerical coin toss
    assert safe.float().mean() > 0.9
    first_bad = (ids.cpu() != ref_ids).float().cumsum(1)
    assert torch.equal(ids.cpu()[first_bad == 0], ref_ids[first_bad == 0])
    assert bool((first_bad[:, -1] == 0).all()) or not bool(safe.all()), "ids diverged although every step had a clear margin"
    if bool((first_bad[:, -1] == 0).all()):
        assert maxerr(lg, ref_lg) < 3e-3
    tcl = F.relu(torch.randn(3, 40, 512, generator=gen(62)))
    ref_dur, ref_raw = R.adm_infer_causal(R.SD(weights_cpu("adm")), tcl, weights.ADM_CFG, return_raw=True)
    dur, raw = ADM.infer_causal(tcl.to(DEV), return_raw=True)
    assert maxerr(raw, ref_raw[..., 0]) < 5e-3
    assert (dur.cpu() != ref_dur).float().mean() < 0.03     # rounding at .5 boundaries only


# ------------------------------------------------------------------ SURVEY.md 8f-2: bulk (ragged) mel extraction
def test_mel_extractor_ragged_batch_vs_oracle():
    """MelSpecExtractor.extract_batch: ragged clips in ONE launch == the oracle clip by clip, truncated to the
    reference's compute_num_frames (modules/tokenizer.py:139-155)."""
    from megatts2_b200.modules.tokenizer import MelSpecExtractor, compute_num_frames
    ex = MelSpecExtractor(DEV)
    lens = [48000, 16000, 5000, 777, 47873, 2816, 2817, 24321]       # incl. lengths on either side of tile / hop edges
    clips = [(torch.rand(n, generator=gen(100 + i)) * 2 - 1) for i, n in enumerate(lens)]
    outs = ex.extract_batch([c.numpy() for c in clips], 16000)
    for c, o, n in zip(clips, outs, lens):
        ref = R.mel_spectrogram(c.unsqueeze(0))[0].transpose(0, 1)[: compute_num_frames(n)]    # (frames, 80)
        assert o.shape == (compute_num_frames(n), 80) == tuple(ref.shape)
        assert float(np.abs(o - ref.numpy()).max()) < 1e-4
        assert float(np.abs(o - ref.numpy()).mean()) < 1e-5
    one = ex.extract(clips[3].numpy(), 16000)                              # single clip == its row of the batch
    assert np.array_equal(one, outs[3])
    with pytest.raises(ValueError):
        ex.extract(np.zeros(512, dtype=np.float32), 16000)                 # reflect padding needs L > n_fft / 2
