"""GPU: duration interpolation.  The mix readout kernel (csrc/ops.cu, adm_readout_mix_kernel) against fp64,
MegaADM.infer_mix against infer and against the fp64 restatement (tests/ref_duration_mix.py), and Megatts.synthesize /
synthesize_stream with duration_weights.

Bars: the readout within READ_TOL = 4e-6 of the fp64 value, relative to the sum of |products| it adds (fp32 accumulation
of D = 768 terms by 32 lanes and a 5-level butterfly: about (D/32 + 5) 2^-24 of that sum); one-weighted-source rows, the
one-hot, K = 1 and replay identities bit for bit; the decode's mixed raw values within RAW_REL = 2e-3 of the fp64 oracle,
relative to max(1, max |raw|) (test_adm_golden's bar on the plain decode), and its durations equal except where the fp64
value lies within 1e-4 of a rounding boundary."""
import numpy as np
import pytest
import torch

import helpers
import ref_duration_mix as DM
from megatts2_b200 import graphs, ops, pack
from megatts2_b200.sampling import Sampling
from oracle import ref_megatts2 as R
from oracle import weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda"
READ_TOL = 4e-6
RAW_REL = 2e-3
NEAR = 1e-4


def gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def tts(weights_cpu):
    return helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)


def weight_patterns(K, B, seed):
    pats = {"one_hot": np.eye(K, dtype=np.float32)[K - 1], "uniform": np.full(K, 1.0, np.float32)}
    if K >= 2:
        pats["0.999/0.001"] = np.array([0.999, 0.001] + [0.0] * (K - 2), np.float32)
        w = np.random.default_rng(seed).random((B, K)).astype(np.float32)
        w[::3, 0] = 0.0                                   # rows with a zero weight, and one-hot rows
        w[1::5] = np.eye(K, dtype=np.float32)[np.arange(len(w[1::5])) % K]
        pats["per_row"] = w
    return pats


# ------------------------------------------------------------------------------ kernel level
@pytest.mark.parametrize("D", [768, 517])
@pytest.mark.parametrize("B", [1, 5, 64])
@pytest.mark.parametrize("K", [1, 2, 3, 8])
def test_readout_mix_against_fp64(K, B, D):
    xl = torch.randn(K, B, D, generator=gen(K * 131 + B * 7 + D))
    wp = torch.randn(D, generator=gen(D)) * 0.05
    worst = 0.0
    for name, w in weight_patterns(K, B, K + B + D).items():
        wr = np.broadcast_to(w, (B, K))
        x = xl.clone()
        for b in range(B):                                  # zero-weight sources predict inf or NaN: ignored
            for k in np.nonzero(wr[b] == 0)[0]:
                x[k, b, (b + k) % D] = float("inf") if (b + k) % 2 else float("nan")
        r, y = ops.adm_readout_mix(x.to(DEV), wp.to(DEV), torch.from_numpy(np.ascontiguousarray(w)))
        r, y = r.cpu(), y.cpu()
        x64, w64 = x.double(), wp.double()
        y64 = x64 @ w64                                     # (K, B)
        scale = x64.abs() @ w64.abs()
        fin = torch.isfinite(y64)
        err = ((y.double() - y64).abs() / scale)[fin]
        worst = max(worst, float(err.max()))
        assert float(err.max()) <= READ_TOL, (name, float(err.max()))
        for b in range(B):
            pos = np.nonzero(wr[b] > 0)[0]
            if len(pos) == 1:                               # one weighted source: its readout, bit for bit
                assert torch.equal(r[b:b + 1].view(torch.int32), y[pos[0], b:b + 1].view(torch.int32)), (name, b)
                continue
            want = DM.mix_readout(y64[:, b], wr[b]).item()
            wn = wr[b] / wr[b][pos].sum(dtype=np.float32)
            bar = READ_TOL * float(sum(wn[k] * scale[k, b] for k in pos)) + 1e-6 * abs(want)
            assert np.isfinite(r[b].item()) and abs(r[b].item() - want) <= bar, (name, b, r[b].item(), want)
    print(f"K={K} B={B} D={D}: max readout error / sum|products| = {worst:.3g}")
    helpers.record("duration_mix_readout", dict(K=K, B=B, D=D, max_rel=worst))


# ------------------------------------------------------------------------------ decode identities
def sources(K, B, T, seed):
    return [torch.randn(B, T, 512, generator=gen(seed + k)).abs().to(DEV) for k in range(K)]


def test_one_hot_mix_equals_infer_on_the_stack(tts):
    adm = tts.adm
    K, B, T = 3, 3, 9
    tcs = sources(K, B, T, 10)
    with graphs.disabled():
        ref_dur, ref_raw = adm.infer(torch.cat(tcs, 0), return_raw=True)
    for k in range(K):
        w = torch.zeros(K)
        w[k] = 0.5
        runs = []
        with graphs.disabled():
            runs.append(adm.infer_mix(tcs, w, return_raw=True))
        for _ in range(3):                                                 # warm-up, capture, replay
            runs.append(adm.infer_mix(tcs, w, return_raw=True))
        blk = slice(k * B, (k + 1) * B)
        for dur, raw, raw_src in runs:
            assert dur.shape == (B, T, 1) and raw_src.shape == (K, B, T)
            assert torch.equal(dur, ref_dur[blk]), k
            assert torch.equal(raw.view(torch.int32), ref_raw[blk].view(torch.int32)), k
            assert torch.equal(raw_src[k], ref_raw[blk]), k


def test_one_source_equals_infer(tts):
    adm = tts.adm
    tc = sources(1, 4, 11, 40)[0]
    ref_dur, ref_raw = adm.infer(tc, return_raw=True)
    for _ in range(3):
        dur, raw, raw_src = adm.infer_mix([tc], [2.0], return_raw=True)
        assert torch.equal(dur, ref_dur) and torch.equal(raw, ref_raw) and torch.equal(raw_src[0], ref_raw)


def test_one_hot_mix_against_infer_on_the_source_alone(tts):
    """B rows instead of K*B: the dense layers may take another tensor-core plan, so raw agrees within rounding and the
    durations are equal away from rounding boundaries."""
    adm = tts.adm
    K, B, T = 2, 8, 24
    tcs = sources(K, B, T, 50)
    for k in range(K):
        w = torch.zeros(K)
        w[k] = 1.0
        dur, raw, _ = adm.infer_mix(tcs, w, return_raw=True)
        ref_dur, ref_raw = adm.infer(tcs[k], return_raw=True)
        err = (raw - ref_raw).abs().max().item()
        assert err <= RAW_REL * max(1.0, ref_raw.abs().max().item()), (k, err)
        near = _boundary_distance(ref_raw.double().cpu()) <= NEAR
        assert torch.equal(dur[..., 0].cpu()[~near], ref_dur[..., 0].cpu()[~near]), k


def test_replay_with_new_weights_needs_no_capture(tts):
    adm = tts.adm
    K, B, T = 2, 4, 10
    tcs = sources(K, B, T, 80)
    for _ in range(2):                                                      # warm-up, capture
        adm.infer_mix(tcs, [0.5, 0.5], return_raw=True)
    n_graphs = len(adm._graphs().cache)
    n_replayed = graphs.replayed_launches
    outs = set()
    for gamma in (0.0, 0.1, 0.5, 0.9, 1.0):
        got = adm.infer_mix(tcs, [1 - gamma, gamma], return_raw=True)
        with graphs.disabled():
            want = adm.infer_mix(tcs, [1 - gamma, gamma], return_raw=True)
        for a, b in zip(got, want):
            assert torch.equal(a, b), gamma
        outs.add(tuple(got[1].flatten().tolist()))
    assert len(adm._graphs().cache) == n_graphs and graphs.replayed_launches > n_replayed
    assert len(outs) == 5                                                   # the weights did change the raw values


def test_graph_replays_after_the_workspace_grew(tts):
    """A mixed decode needs more scratch than the plain one, so switching to it grows the shared workspace.  The plain
    decode's graph, captured on the smaller buffer, must still replay what the eager decode computes, and must not write
    into memory the allocator has since handed to other tensors."""
    adm = tts.adm
    B, T = 5, 7
    tcs = sources(3, B, T, 90)
    with torch.cuda.stream(torch.cuda.Stream()):           # a stream of its own: its workspace starts empty
        with graphs.disabled():
            want = adm.infer(tcs[0], return_raw=True)
        for _ in range(3):                                  # eager, capture, replay on the small workspace
            adm.infer(tcs[0], return_raw=True)
        small = ops.workspace(0, torch.device(DEV)).numel()
        adm.infer_mix(tcs, [0.2, 0.3, 0.5])                 # eager: the workspace grows
        assert ops.workspace(0, torch.device(DEV)).numel() > small
        fill = torch.full((small // 4 + 1024,), 7.0, device=DEV)        # takes freed memory if the old buffer was freed
        got = adm.infer(tcs[0], return_raw=True)
        torch.cuda.synchronize()
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    assert bool((fill == 7.0).all())


# ------------------------------------------------------------------------------ against the fp64 oracle
def _boundary_distance(raw):
    """Distance of raw + 0.5 to the nearest integer: where (raw + 0.5) -> int32 can flip under rounding."""
    x = raw + 0.5
    return (x - x.round()).abs()


@pytest.fixture(scope="module")
def fp64_case(weights_cpu):
    """K = 2, B = 4, T = 20 (up to 160 encoder rows per step, so the tensor-core engines run the dense layers from step 16
    on) and the fp64 oracle's decode of it, computed once for every engine."""
    K, B, T = 2, 4, 20
    tcs = [torch.randn(B, T, 512, generator=gen(900 + k)).abs() for k in range(K)]
    w = np.array([[0.3, 0.7], [1.0, 0.0], [0.0, 2.0], [0.6, 0.4]], np.float32)
    with torch.no_grad():
        dur64, raw64 = DM.adm_infer_mix(DM.sd64(weights_cpu("adm")), [t.double() for t in tcs], weights.ADM_CFG, w,
                                        return_raw=True)[:2]
    return tcs, w, dur64[..., 0], raw64[..., 0]


@pytest.mark.parametrize("engine", [pack.ENGINE_F16X2, pack.ENGINE_BF16X3, pack.ENGINE_FFMA], ids=["f16x2", "bf16x3",
                                                                                                     "ffma"])
def test_infer_mix_against_the_fp64_oracle(tts, fp64_case, engine):
    tcs, w, dur64, raw64 = fp64_case
    with pack.engine_scope(engine):
        dur, raw, _ = tts.adm.infer_mix([t.to(DEV) for t in tcs], w, return_raw=True)
    dur, raw = dur.cpu()[..., 0], raw.cpu().double()
    err = (raw - raw64).abs().max().item()
    scale = max(1.0, raw64.abs().max().item())
    dist = _boundary_distance(raw64)
    near = dist <= NEAR
    print(f"engine {engine}: max |raw - raw_fp64| = {err:.3g} (scale {scale:.3g}); closest boundary "
          f"{dist.min().item():.3g}; {int(near.sum())} of {near.numel()} within {NEAR}")
    helpers.record("duration_mix_vs_fp64", dict(engine=engine, max_abs=err, scale=scale, closest=dist.min().item()))
    assert err <= RAW_REL * scale
    assert torch.equal(dur[~near], dur64[~near])


# ------------------------------------------------------------------------------ end to end
def _e2e_inputs(durations):
    phone = torch.randint(0, 320, (3, 9), generator=gen(61)).to(DEV)
    melp = (torch.randn(3, 56, 80, generator=gen(62)) * 2 - 4).to(DEV)
    pros = [(torch.randn(3, 40, 80, generator=gen(63)) * 2 - 3).to(DEV),
            (torch.randn(3, 72, 80, generator=gen(64)) * 1.5 - 5).to(DEV)]
    forced = torch.full((3, 9), 4, dtype=torch.int32).to(DEV) if durations == "equal" else None
    return phone, melp, pros, forced


W3 = torch.tensor([[0.5, 0.25, 0.25], [0.0, 1.0, 0.0], [0.1, 0.0, 0.9]])
DW3 = torch.tensor([[0.2, 0.3, 0.5], [0.0, 0.0, 1.0], [0.7, 0.3, 0.0]])


@pytest.mark.parametrize("durations", ["equal", "adm"])
def test_synthesize_equals_the_composed_pieces(tts, durations):
    phone, melp, pros, forced = _e2e_inputs(durations)
    smp = dict(sampling=Sampling(temperature=0.9, top_k=50, seed=17), keys=torch.arange(3))
    out = tts.synthesize(phone, melp, forced_durations=forced, prosody_mels=pros, prosody_weights=W3,
                         duration_weights=DW3, return_intermediates=True, **smp)
    with torch.no_grad():
        mrte = tts.generator.mrte
        tc = mrte.tc_latent(phone, melp)
        lats = [mrte.tc_latent(phone, m) for m in pros]
        dt = tts.adm.infer_mix([tc] + lats, DW3)[..., 0]
        d = dt if forced is None else forced
        tce, totals = ops.length_regulate(tc, d, return_host_totals=True)
        srcs = [ops.maxpool_time(tce, 8)] + [
            ops.maxpool_time(ops.length_regulate(lat, d, l_out=tce.shape[1])[0], 8) for lat in lats]
        codes = tts.plm.infer_mix(srcs, W3, **smp)
    assert torch.equal(out["dt"], dt) and torch.equal(out["tc_latent_expand"], tce)
    assert torch.equal(out["p_codes"], codes) and out["totals"] == totals
    # the mixed predictions moved away from the target's own
    assert not torch.equal(tts.adm.infer_mix([tc] + lats, DW3, return_raw=True)[1], tts.adm.infer(tc, return_raw=True)[1])
    if len(set(totals)) == 1:
        with torch.no_grad():
            mel = tts.generator.decode_mel_cl(tce, codes)
            wav = tts.hifi_gan.decode_batch_cl(mel)
        assert torch.equal(out["mel"], mel) and torch.equal(out["wav"], wav)


def test_synthesize_against_the_oracle(weights_cpu, tts):
    """One utterance, K = 2, against the CPU oracle composition: the mixed durations equal the oracle's away from rounding
    boundaries (the frames then use forced durations, as in the prosody-mix oracle test)."""
    phone = torch.randint(0, 320, (1, 9), generator=gen(71))
    melp = torch.randn(1, 72, 80, generator=gen(72)) * 2 - 4
    melq = torch.randn(1, 48, 80, generator=gen(74)) * 2 - 3
    forced = torch.randint(2, 9, (1, 9), generator=gen(73), dtype=torch.int32)
    w = np.array([0.4, 0.6], np.float32)
    out = tts.synthesize(phone.to(DEV), melp.to(DEV), forced_durations=forced.to(DEV), prosody_mels=[melq.to(DEV)],
                         prosody_weights=w, duration_weights=w[::-1].copy(), return_intermediates=True)
    g = R.SD(weights_cpu("g"))
    with torch.no_grad():
        tcs = [R.mrte_tc_latent(g.sub("mrte"), phone, m, weights.G_CFG)[0] for m in (melp, melq)]
        dur, raw = DM.adm_infer_mix(R.SD(weights_cpu("adm")), tcs, weights.ADM_CFG, w[None, ::-1], return_raw=True)[:2]
    near = _boundary_distance(raw[..., 0].double()) <= NEAR
    assert torch.equal(out["dt"].cpu()[~near], dur[..., 0][~near])
    helpers.record("duration_mix_e2e", dict(closest=_boundary_distance(raw.double()).min().item()))


def _run_stream(tts, *args, **kw):
    chunks = list(tts.synthesize_stream(*args, **kw))
    assert chunks[-1]["last"]
    return chunks, torch.cat([c["wav"] for c in chunks], -1)


@pytest.mark.parametrize("durations", ["equal", "adm"])
def test_stream_equals_synthesize(tts, durations):
    phone, melp, pros, forced = _e2e_inputs(durations)
    kw = dict(forced_durations=forced, prosody_mels=pros, prosody_weights=W3, duration_weights=DW3,
              sampling=Sampling(temperature=0.9, top_k=50, seed=17), keys=torch.arange(3, 6))
    ref = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    for cf in (8, max(ref["totals"]) + 100):
        chunks, wav = _run_stream(tts, phone, melp, chunk_frames=cf, **kw)
        assert torch.equal(chunks[-1]["p_codes"], ref["p_codes"]) and torch.equal(chunks[-1]["dt"], ref["dt"])
        assert wav.shape == ref["wav"].shape
        err = (wav - ref["wav"]).abs().max().item()
        assert err <= 1e-5, (cf, err)


def test_range_flag_reruns_on_bf16x3(golden, weights_cpu):
    """The scaled-attention overflow of the prosody-mix range test, with duration_weights: synthesize warns and reruns
    the whole batch - the mixed ADM included - on bf16x3, and equals a bf16x3 run; so does the stream that restarts."""
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
    kw = dict(forced_durations=dur, prosody_mels=pros, prosody_weights=[0.5, 0.5], duration_weights=[0.3, 0.7])
    ops.tc_overflow(torch.device(DEV))
    with pack.engine_scope(pack.ENGINE_F16X2):
        with pytest.warns(UserWarning, match="fp16 range"):
            ref = tts.synthesize(phone, melp, return_intermediates=True, **kw)
        with pytest.warns(UserWarning, match="restarting this stream on the bf16x3 engine"):
            chunks, wav = _run_stream(tts, phone, melp, chunk_frames=1000, **kw)
    with pack.engine_scope(pack.ENGINE_BF16X3):
        want = tts.synthesize(phone, melp, return_intermediates=True, **kw)
        want_dt = tts.adm.infer_mix([want["tc_latent"], tts.generator.mrte.tc_latent(phone, pros[0])], [0.3, 0.7])
    assert torch.equal(ref["dt"], want["dt"]) and torch.equal(want["dt"], want_dt[..., 0])
    assert torch.equal(ref["p_codes"], want["p_codes"]) and torch.equal(ref["wav"], want["wav"])
    assert torch.equal(chunks[-1]["p_codes"], ref["p_codes"]) and torch.equal(chunks[-1]["dt"], ref["dt"])
    assert (wav - ref["wav"]).abs().max().item() <= 1e-5


def test_rejected_combinations(tts):
    from megatts2_b200 import _lib as L
    phone, melp, pros, forced = _e2e_inputs("equal")
    for kw in (dict(prosody_mels=None, prosody_weights=None, duration_weights=[1, 1, 1]),
               dict(causal_decode=True, duration_weights=[1, 1, 1]), dict(duration_weights=[1, 1]),
               dict(duration_weights=[1, -1, 1]), dict(duration_weights=[0, 0, 0]),
               dict(duration_weights=[1, float("nan"), 1]), dict(duration_weights=torch.ones(2, 3))):
        args = dict(prosody_mels=pros, prosody_weights=[1, 1, 1])
        args.update(kw)
        with pytest.raises(L.MttsError):
            tts.synthesize(phone, melp, forced_durations=forced, **args)
    with pytest.raises(L.MttsError):
        tts.synthesize_stream(phone, melp, prosody_mels=pros, prosody_weights=[1, 1, 1], duration_weights=[1, 1])
    with pytest.raises(L.MttsError):
        tts.adm.infer_mix([torch.zeros(2, 4, 512, device=DEV), torch.zeros(2, 5, 512, device=DEV)], [1, 1])
