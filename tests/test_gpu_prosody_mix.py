"""GPU: prosody interpolation.  The mix kernel (csrc/sample.cu, mix_logprob_rows_kernel) against its fp64 oracle
(tests/ref_prosody_mix.py), MegaPLM.infer_mix against infer and against the reference restatement, and
Megatts.synthesize / synthesize_stream with prosody prompts.

Bars: l within MIX_TOL = 2e-5 of the fp64 mixture on tokens with l >= -30 (about seven times the largest error measured,
2.9e-6 on an H100 80GB HBM3 at a 700 W power limit); the
one-weighted-source copy and the non-finite rules exact; picks equal the oracle's except on rows whose two best fp64
scores are within 1e-5 (relative, floor 1), at most 2 per 256 rows; 2^20 draws pass a chi-square test at p >= 1e-6; the
one-hot, K = 1, range and replay identities bit for bit; per-source step logits within test_plm_golden's 2e-3."""
import random

import numpy as np
import pytest
import torch

import helpers
import ref_prosody_mix as PM
from megatts2_b200 import graphs, ops, pack
from megatts2_b200.sampling import Sampling
from oracle import ref_megatts2 as R
from oracle import ref_sampling as RS
from oracle import weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda"
NEAR = 1e-5
MIX_TOL = 2e-5


def gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def tts(weights_cpu):
    return helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)


def weight_patterns(K, B, seed):
    pats = {"one_hot": np.eye(K, dtype=np.float32)[K - 1], "uniform": np.full(K, 1.0, np.float32)}
    if K >= 2:
        pats["0.999/0.001"] = np.array([0.999, 0.001] + [0.0] * (K - 2), np.float32)
        pats["1e-6/1-1e-6"] = np.array([1e-6, 1 - 1e-6] + [0.0] * (K - 2), np.float32)
        w = np.random.default_rng(seed).random((B, K)).astype(np.float32)
        w[::3, 0] = 0.0                                   # rows with a zero weight, and one-hot rows
        w[1::5] = np.eye(K, dtype=np.float32)[np.arange(len(w[1::5])) % K]
        pats["per_row"] = w
    return pats


# ------------------------------------------------------------------------------ kernel level
@pytest.mark.parametrize("V", [1024, 1000, 37])
@pytest.mark.parametrize("K", [1, 2, 3, 8])
def test_mix_kernel_against_fp64(K, V):
    B = 64
    z = torch.randn(K, B, V, generator=gen(K * 7919 + V)) * 3
    worst = 0.0
    for name, w in weight_patterns(K, B, K + V).items():
        got = ops.mix_logprob_rows(z.to(DEV), torch.from_numpy(w)).cpu().numpy().astype(np.float64)
        wr = np.broadcast_to(w, (B, K))
        for b in range(B):
            want = PM.mix_logprobs(z[:, b].numpy(), wr[b])
            if int((wr[b] > 0).sum()) == 1:
                assert np.array_equal(got[b], want), (name, b)        # the raw row, bit for bit
                continue
            m = want >= -30
            err = float(np.abs(got[b][m] - want[m]).max())
            worst = max(worst, err)
            assert err <= MIX_TOL, (name, b, err)
            assert np.all(np.isfinite(got[b]))
    print(f"K={K} V={V}: max |l - l_fp64| = {worst:.3g}")
    helpers.record("prosody_mix_kernel", dict(K=K, V=V, max_abs=worst))


def test_mix_kernel_non_finite_rules():
    V = 64
    z = torch.randn(3, 6, V, generator=gen(5)) * 2
    z[0, 0, :4] = float("nan")                                           # NaN: no mass
    z[1, 1, 7] = float("inf"); z[1, 1, 3] = float("inf")                 # +inf: all mass on index 3
    z[0, 2] = float("nan"); z[2, 2] = -float("inf")                      # sources without a candidate
    z[:, 3] = float("nan")                                               # no candidate at all: -inf, pick 0
    z[0, 4, ::2] = -float("inf")
    z[2, 5] = float("inf")                                               # every index +inf: index 0
    w = torch.tensor([0.5, 0.25, 0.25])
    got = ops.mix_logprob_rows(z.to(DEV), w).cpu().numpy().astype(np.float64)
    for b in range(6):
        want = PM.mix_logprobs(z[:, b].numpy(), w.numpy())
        assert np.array_equal(np.isneginf(got[b]), np.isneginf(want)), b
        assert not np.isnan(got[b]).any() and not np.isposinf(got[b]).any()
        fin = np.isfinite(want)
        assert np.abs(got[b][fin] - want[fin]).max(initial=0.0) <= MIX_TOL, b
    assert np.all(np.isneginf(got[3]))
    smp = Sampling(temperature=0.9, seed=3)
    assert ops.sample_rows(torch.from_numpy(got[3:4]).float().to(DEV), 0, smp, [1]).item() == 0
    assert ops.sample_rows(torch.from_numpy(got[3:4]).float().to(DEV), 0, Sampling(temperature=0.0), [1]).item() == 0
    # one weighted source copies NaN and inf bit for bit
    w1 = torch.tensor([0.0, 2.0, 0.0])
    got1 = ops.mix_logprob_rows(z.to(DEV), w1).cpu()
    assert torch.equal(got1.view(torch.int32), z[1].contiguous().view(torch.int32))


PICKS = [None, (1.0, 0, 1.0), (0.7, 20, 1.0), (1.0, 0, 0.9), (1.3, 50, 0.8)]


@pytest.mark.parametrize("K", [2, 3])
@pytest.mark.parametrize("pi", range(len(PICKS)))
def test_picks_from_the_mixture_agree_with_the_oracle(K, pi):
    rows, V, step = 256, 1024, 11
    z = torch.randn(K, rows, V, generator=gen(300 + 10 * K + pi)) * 3
    w = torch.rand(rows, K, generator=gen(400 + pi)) + 0.05
    keys = torch.randint(0, 2 ** 62, (rows,), generator=gen(500 + pi))
    l = ops.mix_logprob_rows(z.to(DEV), w)
    s = Sampling(temperature=0.0) if PICKS[pi] is None else Sampling(temperature=PICKS[pi][0], top_k=PICKS[pi][1],
                                                                       top_p=PICKS[pi][2], seed=2 ** 63 + 5 * pi)
    got = ops.sample_rows(l, step, s, keys).cpu().numpy()
    smp = None if PICKS[pi] is None else (s.temperature, s.top_k, s.top_p, s.seed)
    bad = 0
    for r in range(rows):
        want, gap = PM.mix_pick(z[:, r].numpy(), w[r].numpy(), step, smp, int(keys[r]))
        if got[r] != want:
            assert gap <= NEAR, (r, gap)
            bad += 1
    print(f"K={K} {PICKS[pi]}: {bad} of {rows} picks differ from the oracle (near-ties)")
    assert bad <= 2


@pytest.mark.parametrize("kw", [dict(temperature=1.0), dict(temperature=0.8, top_k=40), dict(temperature=1.2, top_p=0.9)])
def test_distribution_of_mixed_draws(kw):
    from scipy import stats
    V, n = 1024, 1 << 20
    z = torch.randn(2, 1, V, generator=gen(17)) * 2
    w = torch.tensor([0.3, 0.7])
    l = ops.mix_logprob_rows(z.to(DEV), w)
    s = Sampling(seed=99, **kw)
    got = ops.sample_rows(l.expand(n, V), 4, s, torch.arange(n)).cpu().numpy()
    obs = np.bincount(got, minlength=V).astype(np.float64)
    lo = PM.mix_logprobs(z[:, 0].numpy(), w.numpy()).astype(np.float32)
    p = RS.target_distribution(lo, s.temperature, s.top_k, s.top_p)
    exp = n * p
    big = exp >= 5
    o = np.append(obs[big], obs[~big].sum())
    e = np.append(exp[big], exp[~big].sum())
    if e[-1] == 0:
        assert o[-1] == 0
        o, e = o[:-1], e[:-1]
    res = stats.chisquare(o, e * (o.sum() / e.sum()))
    print(f"{kw}: chi2 {res.statistic:.1f} over {len(o) - 1} dof, p-value {res.pvalue:.3g}")
    assert res.pvalue >= 1e-6


# ------------------------------------------------------------------------------ decode identities
SAMPLINGS = [None, Sampling(temperature=0.8, top_k=20, seed=5), Sampling(temperature=1.3, top_p=0.9, seed=2 ** 63 + 11)]


def sources(K, B, T, dim, seed):
    return [torch.randn(B, T, dim, generator=gen(seed + k)).abs().to(DEV) for k in range(K)]


@pytest.mark.parametrize("smp", range(len(SAMPLINGS)))
def test_one_hot_mix_equals_infer_on_the_stack(tts, smp):
    plm, sampling = tts.plm, SAMPLINGS[smp]
    K, B, T = 3, 3, 9
    tcs = sources(K, B, T, plm.tc_latent_dim, 10 + smp)
    keys = torch.arange(7, 7 + B, dtype=torch.int64)
    kw = {} if sampling is None else dict(sampling=sampling)
    with graphs.disabled():
        ref_codes, ref_logits = plm.infer(torch.cat(tcs, 0), return_logits=True,
                                          **(dict(kw, keys=keys.repeat(K)) if kw else {}))
    for k in range(K):
        w = torch.zeros(K)
        w[k] = 0.5
        runs = []
        with graphs.disabled():
            runs.append(plm.infer_mix(tcs, w, return_logits=True, keys=keys, **kw))
        for _ in range(3):                                                 # warm-up, capture, replay
            runs.append(plm.infer_mix(tcs, w, return_logits=True, keys=keys, **kw))
        for codes, logits in runs:
            assert logits.shape == (K, B, T, plm.vq_bins)
            assert torch.equal(codes, ref_codes[k * B:(k + 1) * B]), k
            assert torch.equal(logits[k], ref_logits[k * B:(k + 1) * B]), k


@pytest.mark.parametrize("smp", range(len(SAMPLINGS)))
def test_one_source_equals_infer(tts, smp):
    plm, sampling = tts.plm, SAMPLINGS[smp]
    tc = sources(1, 4, 11, plm.tc_latent_dim, 40 + smp)[0]
    kw = {} if sampling is None else dict(sampling=sampling, keys=torch.arange(4) * 3)
    ref = plm.infer(tc, return_logits=True, **kw)
    for _ in range(3):
        codes, logits = plm.infer_mix([tc], [2.0], return_logits=True, **kw)
        assert torch.equal(codes, ref[0]) and torch.equal(logits[0], ref[1])


@pytest.mark.parametrize("smp", range(len(SAMPLINGS)))
def test_mixed_ranges_equal_the_whole_decode(tts, smp):
    plm, sampling = tts.plm, SAMPLINGS[smp]
    K, B, T = 2, 3, 13
    tcs = sources(K, B, T, plm.tc_latent_dim, 60 + smp)
    w = torch.tensor([[0.5, 0.5], [0.2, 0.8], [1.0, 0.0]])
    kw = {} if sampling is None else dict(sampling=sampling, keys=torch.arange(3, 3 + B))
    with graphs.disabled():
        ref_codes, ref_logits = plm.infer_mix(tcs, w, return_logits=True, **kw)
    rng = random.Random(smp)
    cut_sets = [[0, T], list(range(T + 1)), [0] + sorted(rng.sample(range(1, T), 3)) + [T]]
    for graphed in (False, True):
        for cuts in cut_sets:
            for rep in range(3 if graphed else 1):
                dec = plm.begin_decode(tcs, weights=w, **kw)
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
                assert torch.equal(torch.cat(logits, 2), ref_logits), (graphed, cuts, rep)
                assert torch.equal(dec.codes, ref_codes)


def test_replay_with_new_weights_needs_no_capture(tts):
    plm = tts.plm
    K, B, T = 2, 4, 10
    tcs = sources(K, B, T, plm.tc_latent_dim, 80)
    smp = Sampling(temperature=0.9, top_k=30, seed=4)
    for _ in range(2):                                                      # warm-up, capture
        plm.infer_mix(tcs, [0.5, 0.5], sampling=smp)
    n_graphs = len(plm._graphs().cache)
    n_replayed = graphs.replayed_launches
    outs = set()
    for gamma in (0.0, 0.1, 0.5, 0.9, 1.0):
        for s in (smp, Sampling(temperature=0.9, top_k=30, seed=1234)):    # a new seed is a device input too
            got = plm.infer_mix(tcs, [1 - gamma, gamma], sampling=s)
            with graphs.disabled():
                want = plm.infer_mix(tcs, [1 - gamma, gamma], sampling=s)
            assert torch.equal(got, want), (gamma, s.seed)
            outs.add(tuple(got.flatten().tolist()))
    assert len(plm._graphs().cache) == n_graphs and graphs.replayed_launches > n_replayed
    assert len(outs) > 2                                                    # the weights did change the codes


# ------------------------------------------------------------------------------ against the reference
@pytest.mark.parametrize("K", [2, 3])
def test_infer_mix_against_the_reference(weights_cpu, tts, K):
    plm, sd, cfg = tts.plm, R.SD(weights_cpu("plm")), weights.PLM_CFG
    B, T = 2, 12
    tcs = [torch.randn(B, T, plm.tc_latent_dim, generator=gen(900 + k)).abs() for k in range(K)]
    w = np.full(K, 0.5, np.float32) if K == 2 else np.array([0.2, 0.5, 0.3], np.float32)
    codes, logits = plm.infer_mix([t.to(DEV) for t in tcs], w, return_logits=True)
    codes, logits = codes.cpu(), logits.cpu()
    prefix = torch.cat([torch.full((B, 1), cfg["vq_bins"], dtype=torch.int64), codes], 1)
    worst = 0.0
    for t in range(T):
        for k in range(K):
            ref = R.plm_step_logits(sd, tcs[k], prefix[:, :t + 1], cfg)
            err = (logits[k, :, t] - ref).abs().max().item()
            worst = max(worst, err)
            assert err <= 2e-3, (t, k, err)
        for b in range(B):
            pick, gap = PM.mix_pick(logits[:, b, t].numpy(), w)
            assert pick == int(codes[b, t]) or gap <= NEAR, (t, b, gap)
    helpers.record("prosody_mix_step_logits", dict(K=K, max_abs=worst))
    # free-running: equal up to the first near-tie of the oracle
    o_codes, _, gaps = PM.plm_infer_mix(sd, tcs, cfg, np.broadcast_to(w, (B, K)), return_logits=True)
    for b in range(B):
        for t in range(T):
            if gaps[b, t] <= NEAR:
                break
            assert int(o_codes[b, t]) == int(codes[b, t]), (b, t)


# ------------------------------------------------------------------------------ end to end
def _e2e_inputs(durations):
    phone = torch.randint(0, 320, (3, 9), generator=gen(61)).to(DEV)
    melp = (torch.randn(3, 56, 80, generator=gen(62)) * 2 - 4).to(DEV)
    pros = [(torch.randn(3, 40, 80, generator=gen(63)) * 2 - 3).to(DEV),
            (torch.randn(3, 72, 80, generator=gen(64)) * 1.5 - 5).to(DEV)]
    forced = (torch.full((3, 9), 4, dtype=torch.int32) if durations == "equal" else
              torch.randint(1, 7, (3, 9), generator=gen(65), dtype=torch.int32)).to(DEV)
    return phone, melp, pros, (None if durations == "adm" else forced)


W3 = torch.tensor([[0.5, 0.25, 0.25], [0.0, 1.0, 0.0], [0.1, 0.0, 0.9]])


def test_synthesize_equals_the_composed_pieces(tts):
    phone, melp, pros, forced = _e2e_inputs("equal")
    smp = dict(sampling=Sampling(temperature=0.9, top_k=50, seed=17), keys=torch.arange(3))
    out = tts.synthesize(phone, melp, forced_durations=forced, prosody_mels=pros, prosody_weights=W3,
                         return_intermediates=True, **smp)
    with torch.no_grad():
        mrte = tts.generator.mrte
        tc = mrte.tc_latent(phone, melp)
        dt = tts.adm.infer(tc)[..., 0]
        d = forced
        tce, _ = ops.length_regulate(tc, d, return_host_totals=True)
        srcs = [ops.maxpool_time(tce, 8)] + [
            ops.maxpool_time(ops.length_regulate(mrte.tc_latent(phone, m), d, l_out=tce.shape[1])[0], 8) for m in pros]
        codes = tts.plm.infer_mix(srcs, W3, **smp)
        mel = tts.generator.decode_mel_cl(tce, codes)
        wav = tts.hifi_gan.decode_batch_cl(mel)
    assert torch.equal(out["p_codes"], codes) and torch.equal(out["dt"], dt)
    assert torch.equal(out["mel"], mel) and torch.equal(out["wav"], wav)


def test_synthesize_against_the_oracle(weights_cpu, tts):
    """One utterance, K = 2, against the CPU oracle composition: ids up to the first near-tie, mel L1 <= 1e-4."""
    phone = torch.randint(0, 320, (1, 9), generator=gen(71))
    melp = torch.randn(1, 72, 80, generator=gen(72)) * 2 - 4
    melq = torch.randn(1, 48, 80, generator=gen(74)) * 2 - 3
    forced = torch.randint(2, 9, (1, 9), generator=gen(73), dtype=torch.int32)
    w = np.array([0.4, 0.6], np.float32)
    out = tts.synthesize(phone.to(DEV), melp.to(DEV), forced_durations=forced.to(DEV), prosody_mels=[melq.to(DEV)],
                         prosody_weights=w, return_intermediates=True)
    g = R.SD(weights_cpu("g"))
    with torch.no_grad():
        tcs = []
        for m in (melp, melq):
            tc, _, _ = R.mrte_tc_latent(g.sub("mrte"), phone, m, weights.G_CFG)
            tce = R.length_regulate(tc, forced)
            tcs.append(torch.nn.functional.max_pool1d(tce.transpose(1, 2), 8, ceil_mode=True).transpose(1, 2))
            if m is melp:
                tce0 = tce
        codes, _, gaps = PM.plm_infer_mix(R.SD(weights_cpu("plm")), tcs, weights.PLM_CFG, w[None], return_logits=True)
    T = codes.shape[1]
    first_tie = next((t for t in range(T) if gaps[0, t] <= NEAR), T)
    assert torch.equal(out["p_codes"][:, :first_tie].cpu(), codes[:, :first_tie])
    if first_tie == T:
        mel = R.mel_decode(g, tce0, codes, weights.G_CFG)
        t = int(forced.sum())
        err = (out["mel"][:, :t].cpu() - mel.transpose(1, 2)).abs().mean().item()
        helpers.record("prosody_mix_e2e_mel_l1", dict(mean_abs=err))
        assert err <= 1e-4


def _run_stream(tts, *args, **kw):
    chunks = list(tts.synthesize_stream(*args, **kw))
    assert chunks[-1]["last"]
    return chunks, torch.cat([c["wav"] for c in chunks], -1)


@pytest.mark.parametrize("durations", ["equal", "ragged"])
@pytest.mark.parametrize("prompt", [False, True])
def test_stream_equals_synthesize(tts, durations, prompt):
    phone, melp, pros, forced = _e2e_inputs(durations)
    kw = dict(forced_durations=forced, prompt_mels=melp if prompt else None, prosody_mels=pros, prosody_weights=W3,
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


def test_range_flag_reruns_on_bf16x3(golden, weights_cpu):
    """The scaled-attention overflow of test_stream_range_flag_restarts_on_bf16x3, with a prosody prompt: synthesize
    warns and reruns on bf16x3, and equals a bf16x3 run; so does the stream that restarts."""
    g = golden("e2e")
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    phone = torch.randint(0, 320, (1, 70), generator=gen(13)).to(DEV)
    dur = torch.full((1, 70), 8, dtype=torch.int32, device=DEV)
    melp = g["mel_prompt"].to(DEV)
    pros = [(torch.randn(1, 64, 80, generator=gen(14)) * 2 - 4).to(DEV)]
    lyr = tts.plm.plm.layers[0]
    with torch.no_grad():
        lyr.attn.w_q.weight.mul_(2.0 ** 17)
        lyr.attn.w_k.weight.mul_(2.0 ** -17)
    kw = dict(forced_durations=dur, prosody_mels=pros, prosody_weights=[0.5, 0.5])
    ops.tc_overflow(torch.device(DEV))
    with pack.engine_scope(pack.ENGINE_F16X2):
        with pytest.warns(UserWarning, match="fp16 range"):
            ref = tts.synthesize(phone, melp, return_intermediates=True, **kw)
        with pytest.warns(UserWarning, match="restarting this stream on the bf16x3 engine"):
            chunks, wav = _run_stream(tts, phone, melp, chunk_frames=1000, **kw)
    with pack.engine_scope(pack.ENGINE_BF16X3):
        want = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    assert torch.equal(ref["p_codes"], want["p_codes"]) and torch.equal(ref["wav"], want["wav"])
    assert torch.equal(chunks[-1]["p_codes"], ref["p_codes"]) and (wav - ref["wav"]).abs().max().item() <= 1e-5


def test_rejected_combinations(tts):
    from megatts2_b200 import _lib as L
    phone, melp, pros, forced = _e2e_inputs("equal")
    for kw in (dict(causal_decode=True, prosody_weights=[1, 1, 1]), dict(prosody_weights=[1, 1]),
               dict(prosody_weights=[1, -1, 1]), dict(prosody_weights=[0, 0, 0]),
               dict(prosody_weights=[1, float("nan"), 1]), dict(prosody_weights=torch.ones(2, 3))):
        with pytest.raises(L.MttsError):
            tts.synthesize(phone, melp, forced_durations=forced, prosody_mels=pros, **kw)
    with pytest.raises(L.MttsError):
        tts.synthesize(phone, melp, prosody_mels=[pros[0][:2]], prosody_weights=[1, 1])
    with pytest.raises(L.MttsError):
        tts.synthesize(phone, melp, prosody_mels=[pros[0]] * 8, prosody_weights=[1] * 9)
    with pytest.raises(L.MttsError):
        tts.synthesize_many([(phone[0], melp[0])], prosody_mels=pros, prosody_weights=[1, 1, 1])
    with pytest.raises(L.MttsError):
        tts.synthesize_stream(phone, melp, prosody_mels=pros, prosody_weights=[1, 1])
    with pytest.raises(L.MttsError):
        tts.plm.infer_mix([torch.zeros(2, 4, 512, device=DEV), torch.zeros(2, 5, 512, device=DEV)], [1, 1])
