"""GPU: mix schedules - prosody and duration weights that change along the utterance.  The phone -> step expansion kernel
(csrc/ops.cu, mix_step_weights_kernel) against the host rule (tests/ref_mix_schedule.py), MegaPLM.infer_mix /
begin_decode and MegaADM.infer_mix with (B, T, K) weights against the per-utterance mix and the fp64 restatement, and
Megatts.synthesize / synthesize_stream with per-phone weights.

Bars: the expansion bit for bit; a schedule that repeats one row per utterance (materialised, or w_st = 0) equals the
(B, K) mix bit for bit; the mixed l of a step within MIX_TOL = 2e-5 of the fp64 mixture of the decode's own per-source
logits (test_gpu_prosody_mix's bar) and picks equal except on fp64 near-ties (relative gap <= 1e-5); per-source logits
within test_plm_golden's 2e-3 of the reference; the ADM's mixed readout within READ_TOL = 4e-6 of the fp64 mix of its own
per-source readouts, relative to sum_k w^_k |y_k| (test_gpu_duration_mix's bar), its raw values within RAW_REL = 2e-3 of the
fp64 oracle and durations equal except within 1e-4 of a rounding boundary; a one-hot step gives that source's raw row or
readout exactly; ranges, replays and synthesize against the composed pieces bit for bit; the stream within 1e-5."""
import contextlib
import ctypes as C
import random

import numpy as np
import pytest
import torch

import helpers
import ref_duration_mix as DM
import ref_mix_schedule as MS
import ref_prosody_mix as PM
from megatts2_b200 import _lib as L
from megatts2_b200 import graphs, ops, pack
from megatts2_b200.sampling import Sampling
from oracle import ref_megatts2 as R
from oracle import weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda"
NEAR = 1e-5
MIX_TOL = 2e-5
READ_TOL = 4e-6
RAW_REL = 2e-3
ROUND_NEAR = 1e-4
ENGINES = pytest.mark.parametrize("engine", [pack.ENGINE_F16X2, pack.ENGINE_BF16X3, pack.ENGINE_FFMA],
                                  ids=["f16x2", "bf16x3", "ffma"])


def gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def tts(weights_cpu):
    return helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)


def sources(K, B, T, seed):
    return [torch.randn(B, T, 512, generator=gen(seed + k)).abs().to(DEV) for k in range(K)]


def schedule(B, T, K, seed):
    """Rows of every kind: random positive rows, rows with zeros, one-hot rows and, in utterance 1, a piecewise one-hot
    schedule that switches source every few steps."""
    rng = np.random.default_rng(seed)
    w = rng.random((B, T, K)).astype(np.float32) + np.float32(0.05)
    w[0, ::3, 0] = 0.0
    w[0, 1::4] = np.eye(K, dtype=np.float32)[np.arange(len(w[0, 1::4])) % K]
    if B > 1:
        w[1] = np.eye(K, dtype=np.float32)[(np.arange(T) // 3) % K] * np.float32(0.75)
    return w


# ------------------------------------------------------------------------------ the expansion kernel
def _expand_case(durations, K, T, seed):
    d = np.asarray(durations, dtype=np.int32)
    B, Tp = d.shape
    pw = np.random.default_rng(seed).random((B, Tp, K)).astype(np.float32)
    pw.reshape(-1)[::7] = -0.0                          # the copy is of bits: -0 and NaN payloads survive it
    pw.reshape(-1)[3::11] = np.float32("nan")
    got = ops.mix_step_weights(torch.from_numpy(pw).to(DEV), torch.from_numpy(d).to(DEV), T).cpu()
    want = torch.from_numpy(np.ascontiguousarray(MS.step_weights(pw, d, T)))
    assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (durations if d.size < 64 else (B, Tp), T)


@pytest.mark.parametrize("durations, T", [
    ([[8, 8]], 2), ([[4, 4, 8]], 2), ([[2, 3, 3, 8]], 2), ([[5, 0, 0, 11]], 2), ([[0, 8, 0]], 3), ([[4, 6, 0, 0]], 4),
    ([[0, 0, 0]], 2), ([[-3, 8, -1]], 2), ([[13]], 3), ([[8, 8, 8], [20, 0, 1]], 3), ([[1] * 8 + [2, 6]], 2),
    ([[3, 4]], 0), ([[7, 9, 1]], 1),
])
@pytest.mark.parametrize("K", [1, 3, 8])
def test_expansion_edge_cases(durations, T, K):
    _expand_case(durations, K, T, K)


@pytest.mark.parametrize("Tp", [1, 7, 255, 257, 1000, 8192])
def test_expansion_random_durations(Tp):
    rng = np.random.default_rng(Tp)
    B = 64 if Tp < 1000 else 3
    d = rng.integers(0, 14, (B, Tp))
    d[rng.random((B, Tp)) < 0.15] = 0
    d[0, :] = 0                                         # L = 0
    d[1 % B, Tp // 2:] = 0                              # a silent tail
    T = int(-(-d.sum(1).max() // 8)) + 2                # ragged totals, and steps past every end
    _expand_case(d, 2, T, Tp)


# ------------------------------------------------------------------------------ identities with the per-utterance mix
SAMPLINGS = [None, Sampling(temperature=0.8, top_k=20, seed=5)]


def _plm_steps_direct(plm, tcs, w, w_sb, w_st, sampling, keys):
    """mtts_plm_infer_mix_steps_f32 called with explicit weight strides -> (codes, logits (K, B, T, V))."""
    K, (B, T, _) = len(tcs), tcs[0].shape
    tc = torch.cat(tcs, 0)
    pl = plm._plan_get(tc.device, T)
    lib = L.lib()
    m = C.byref(pl.struct)
    codes = torch.empty(B, T, dtype=torch.int64, device=DEV)
    logits = torch.empty(K * B, T, plm.vq_bins, device=DEV)
    nbytes = lib.mtts_plm_infer_mix_workspace_bytes(m, K, B, T)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    smp = None if sampling is None else (sampling.seed_tensor(DEV), keys.to(DEV))
    s = None if sampling is None else C.byref(sampling.struct(*smp))
    L.check(lib.mtts_plm_infer_mix_steps_f32(m, K, tc.data_ptr(), tc.stride(0), tc.stride(1), B, T, w.data_ptr(), w_sb,
                                             w_st, codes.data_ptr(), logits.data_ptr(), s, ws.data_ptr(), nbytes,
                                             ops._stream()))
    torch.cuda.synchronize()
    return codes, logits.reshape(K, B, T, -1)


@pytest.mark.parametrize("smp", range(len(SAMPLINGS)))
def test_constant_plm_schedule_equals_the_row_mix(tts, smp):
    plm, sampling = tts.plm, SAMPLINGS[smp]
    K, B, T = 3, 4, 11
    tcs = sources(K, B, T, 10 + smp)
    w = torch.from_numpy(schedule(B, 1, K, 3)[:, 0])
    kw = {} if sampling is None else dict(sampling=sampling, keys=torch.arange(5, 5 + B))
    with graphs.disabled():
        ref_codes, ref_logits = plm.infer_mix(tcs, w, return_logits=True, **kw)
    sched = w[:, None, :].expand(B, T, K)
    for rep in range(4):                                # eager, warm-up, capture, replay
        with graphs.disabled() if rep == 0 else contextlib.nullcontext():
            codes, logits = plm.infer_mix(tcs, sched, return_logits=True, **kw)
        assert torch.equal(codes, ref_codes) and torch.equal(logits, ref_logits), rep
    codes, logits = _plm_steps_direct(plm, tcs, w.to(DEV), K, 0, sampling, kw.get("keys"))   # w_st = 0
    assert torch.equal(codes, ref_codes) and torch.equal(logits, ref_logits)


def test_constant_adm_schedule_equals_the_row_mix(tts):
    adm = tts.adm
    K, B, T = 3, 4, 13
    tcs = sources(K, B, T, 30)
    w = torch.from_numpy(schedule(B, 1, K, 4)[:, 0])
    with graphs.disabled():
        ref = adm.infer_mix(tcs, w, return_raw=True)
    for rep in range(4):
        with graphs.disabled() if rep == 0 else contextlib.nullcontext():
            got = adm.infer_mix(tcs, w[:, None, :].expand(B, T, K), return_raw=True)
        for a, b in zip(got, ref):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), rep
    # w_st = 0 through the C entry
    tc = torch.cat(tcs, 0)
    pl = adm._plan_get(tc.device, T)
    lib, m = L.lib(), C.byref(pl.struct)
    dur = torch.empty(B, T, dtype=torch.int32, device=DEV)
    raw = torch.empty(B, T, device=DEV)
    nbytes = lib.mtts_adm_infer_mix_workspace_bytes(m, K, B, T)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    wd = w.to(DEV)
    L.check(lib.mtts_adm_infer_mix_steps_f32(m, K, tc.data_ptr(), tc.stride(0), tc.stride(1), B, T, wd.data_ptr(), K, 0,
                                             dur.data_ptr(), raw.data_ptr(), None, ws.data_ptr(), nbytes, ops._stream()))
    torch.cuda.synchronize()
    assert torch.equal(dur, ref[0][..., 0]) and torch.equal(raw.view(torch.int32), ref[1].view(torch.int32))


# ------------------------------------------------------------------------------ schedules against fp64
@pytest.fixture(scope="module")
def plm_case(weights_cpu):
    K, B, T = 2, 3, 12
    tcs = [torch.randn(B, T, 512, generator=gen(700 + k)).abs() for k in range(K)]
    w = schedule(B, T, K, 7)
    with torch.no_grad():
        o_codes, _, gaps = MS.plm_infer_mix_steps(R.SD(weights_cpu("plm")), tcs, weights.PLM_CFG, w, return_logits=True)
    return tcs, w, o_codes, gaps


@ENGINES
def test_plm_schedule_against_fp64(weights_cpu, tts, plm_case, engine):
    plm, sd, cfg = tts.plm, R.SD(weights_cpu("plm")), weights.PLM_CFG
    tcs, w, o_codes, gaps = plm_case
    K, (B, T, _) = len(tcs), tcs[0].shape
    with pack.engine_scope(engine):
        codes, logits = plm.infer_mix([t.to(DEV) for t in tcs], w, return_logits=True)
    prefix = torch.cat([torch.full((B, 1), cfg["vq_bins"], dtype=torch.int64), codes.cpu()], 1)
    worst_l = worst_z = 0.0
    for t in range(T):
        l_gpu = ops.mix_logprob_rows(logits[:, :, t], torch.from_numpy(w[:, t])).cpu().numpy().astype(np.float64)
        lg = logits[:, :, t].cpu()
        for k in range(K):
            ref = R.plm_step_logits(sd, tcs[k], prefix[:, :t + 1], cfg)
            worst_z = max(worst_z, (lg[k] - ref).abs().max().item())
        for b in range(B):
            pos = np.nonzero(w[b, t] > 0)[0]
            if len(pos) == 1:                            # a one-hot step: that source's raw row decides, exactly
                assert int(codes[b, t]) == int(torch.argmax(lg[pos[0], b])), (b, t)
                continue
            want = PM.mix_logprobs(lg[:, b].numpy(), w[b, t])
            m = want >= -30
            worst_l = max(worst_l, float(np.abs(l_gpu[b][m] - want[m]).max()))
            pick, gap = PM.mix_pick(lg[:, b].numpy(), w[b, t], t)
            assert pick == int(codes[b, t]) or gap <= NEAR, (b, t, gap)
    print(f"engine {engine}: max |l - l_fp64| = {worst_l:.3g}, max |z - z_ref| = {worst_z:.3g}")
    helpers.record("mix_schedule_plm", dict(engine=engine, max_l=worst_l, max_logit=worst_z))
    assert worst_l <= MIX_TOL and worst_z <= 2e-3
    for b in range(B):                                   # free-running: equal up to the oracle's first near-tie
        for t in range(T):
            if gaps[b, t] <= NEAR:
                break
            assert int(o_codes[b, t]) == int(codes[b, t]), (b, t)


@pytest.fixture(scope="module")
def adm_case(weights_cpu):
    K, B, T = 2, 4, 20
    tcs = [torch.randn(B, T, 512, generator=gen(900 + k)).abs() for k in range(K)]
    w = schedule(B, T, K, 9)
    with torch.no_grad():
        dur64, raw64 = MS.adm_infer_mix_steps(DM.sd64(weights_cpu("adm")), [t.double() for t in tcs], weights.ADM_CFG, w)
    return tcs, w, dur64, raw64


@ENGINES
def test_adm_schedule_against_fp64(tts, adm_case, engine):
    tcs, w, dur64, raw64 = adm_case
    K, (B, T, _) = len(tcs), tcs[0].shape
    with pack.engine_scope(engine):
        dur, raw, y = tts.adm.infer_mix([t.to(DEV) for t in tcs], w, return_raw=True)
    dur, raw, y = dur.cpu()[..., 0], raw.cpu(), y.cpu()
    worst = 0.0
    for b in range(B):
        for t in range(T):
            pos = np.nonzero(w[b, t] > 0)[0]
            if len(pos) == 1:                            # a one-hot step feeds back that source's readout, bit for bit
                assert raw[b, t].view(torch.int32) == y[pos[0], b, t].view(torch.int32), (b, t)
                continue
            want = DM.mix_readout(y[:, b, t].double(), w[b, t]).item()
            wn = w[b, t] / w[b, t][pos].sum(dtype=np.float32)
            scale = float(sum(wn[k] * abs(y[k, b, t].item()) for k in pos))
            worst = max(worst, abs(raw[b, t].item() - want) / max(scale, 1e-30))
            assert abs(raw[b, t].item() - want) <= READ_TOL * scale + 1e-6 * abs(want), (b, t)
    err = (raw.double() - raw64).abs().max().item()
    scale = max(1.0, raw64.abs().max().item())
    x = raw64 + 0.5
    near = (x - x.round()).abs() <= ROUND_NEAR
    print(f"engine {engine}: readout rel err {worst:.3g}; max |raw - raw_fp64| = {err:.3g}; {int(near.sum())} near")
    helpers.record("mix_schedule_adm", dict(engine=engine, readout_rel=worst, max_abs=err, scale=scale))
    assert err <= RAW_REL * scale
    assert torch.equal(dur[~near], dur64[~near])


# ------------------------------------------------------------------------------ ranges and replays
@pytest.mark.parametrize("smp", range(len(SAMPLINGS)))
def test_schedule_ranges_equal_the_whole_decode(tts, smp):
    plm, sampling = tts.plm, SAMPLINGS[smp]
    K, B, T = 3, 3, 13
    tcs = sources(K, B, T, 60 + smp)
    w = torch.from_numpy(schedule(B, T, K, 60 + smp))
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
                    with contextlib.nullcontext() if graphed else graphs.disabled():
                        c, lg = plm.decode_until(dec, t1, return_logits=True)
                    codes.append(c)
                    logits.append(lg)
                assert torch.equal(torch.cat(codes, 1), ref_codes), (graphed, cuts, rep)
                assert torch.equal(torch.cat(logits, 2), ref_logits), (graphed, cuts, rep)


def test_replay_with_new_schedules_needs_no_capture(tts):
    plm, adm = tts.plm, tts.adm
    K, B, T = 2, 4, 10
    tcs = sources(K, B, T, 80)
    first = torch.from_numpy(schedule(B, T, K, 0))
    for _ in range(2):                                  # warm-up, capture
        plm.infer_mix(tcs, first)
        adm.infer_mix(tcs, first, return_raw=True)
        plm.decode_until(plm.begin_decode(tcs, weights=first), T)
    n_graphs = (len(plm._graphs().cache), len(plm._graphs("range").cache), len(adm._graphs().cache))
    n_replayed = graphs.replayed_launches
    outs = set()
    for seed in range(1, 5):
        w = torch.from_numpy(schedule(B, T, K, seed))
        got = (plm.infer_mix(tcs, w), adm.infer_mix(tcs, w, return_raw=True)[1],
               plm.decode_until(plm.begin_decode(tcs, weights=w), T))
        with graphs.disabled():
            want = (plm.infer_mix(tcs, w), adm.infer_mix(tcs, w, return_raw=True)[1],
                    plm.decode_until(plm.begin_decode(tcs, weights=w), T))
        for a, b in zip(got, want):
            assert torch.equal(a, b), seed
        assert torch.equal(got[0], got[2])
        outs.add(tuple(got[1].flatten().tolist()))
    assert (len(plm._graphs().cache), len(plm._graphs("range").cache), len(adm._graphs().cache)) == n_graphs
    assert graphs.replayed_launches > n_replayed and len(outs) == 4


# ------------------------------------------------------------------------------ end to end
def _e2e_inputs(durations):
    phone = torch.randint(0, 320, (3, 9), generator=gen(61)).to(DEV)
    melp = (torch.randn(3, 56, 80, generator=gen(62)) * 2 - 4).to(DEV)
    pros = [(torch.randn(3, 40, 80, generator=gen(63)) * 2 - 3).to(DEV),
            (torch.randn(3, 72, 80, generator=gen(64)) * 1.5 - 5).to(DEV)]
    forced = (None if durations == "adm" else torch.full((3, 9), 4, dtype=torch.int32) if durations == "equal" else
              torch.tensor([[4, 0, 9, 3, 1, 8, 2, 6, 5], [1, 1, 1, 1, 1, 1, 1, 1, 16], [7] * 9], dtype=torch.int32))
    return phone, melp, pros, None if forced is None else forced.to(DEV)


W3 = torch.tensor([[0.5, 0.25, 0.25], [0.0, 1.0, 0.0], [0.1, 0.0, 0.9]])
DW3 = torch.tensor([[0.2, 0.3, 0.5], [0.0, 0.0, 1.0], [0.7, 0.3, 0.0]])
SMP = dict(sampling=Sampling(temperature=0.9, top_k=50, seed=17), keys=torch.arange(3))


@pytest.mark.parametrize("durations", ["adm", "ragged"])
def test_constant_per_phone_weights_equal_the_row_weights(tts, durations):
    phone, melp, pros, forced = _e2e_inputs(durations)
    Tp = phone.shape[1]
    kw = dict(forced_durations=forced, prosody_mels=pros, return_intermediates=True, **SMP)
    ref = tts.synthesize(phone, melp, prosody_weights=W3, duration_weights=DW3, **kw)
    got = tts.synthesize(phone, melp, prosody_weights=W3[:, None].expand(3, Tp, 3),
                         duration_weights=DW3[:, None].expand(3, Tp, 3), **kw)
    assert torch.equal(got["p_codes"], ref["p_codes"]) and torch.equal(got["dt"], ref["dt"])
    assert torch.equal(got["wav"], ref["wav"]) and got["wav_lens"] == ref["wav_lens"]
    T = ref["p_codes"].shape[1]
    assert torch.equal(got["prosody_step_weights"].cpu(), W3[:, None].expand(3, T, 3))
    assert "prosody_step_weights" not in ref


def _phone_schedules(Tp):
    pw = torch.zeros(3, Tp, 3)
    pw[0, :Tp // 2, 1] = 1.0                            # the first half like prompt 1, the rest like prompt 2
    pw[0, Tp // 2:, 2] = 1.0
    pw[1] = torch.linspace(0, 1, Tp)[:, None] * torch.tensor([-1.0, 0.0, 1.0]) + torch.tensor([1.0, 0.0, 0.0])
    pw[2] = torch.rand(Tp, 3, generator=gen(5)) + 0.05  # a glide from the target to prompt 2; random rows
    dw = pw.flip(-1).clone()
    return pw, dw


@pytest.mark.parametrize("durations", ["adm", "equal", "ragged"])
def test_per_phone_schedule_equals_the_composed_pieces(tts, durations):
    phone, melp, pros, forced = _e2e_inputs(durations)
    pw, dw = _phone_schedules(phone.shape[1])
    out = tts.synthesize(phone, melp, forced_durations=forced, prosody_mels=pros, prosody_weights=pw,
                         duration_weights=dw, return_intermediates=True, **SMP)
    with torch.no_grad():
        mrte = tts.generator.mrte
        tc = mrte.tc_latent(phone, melp)
        lats = [mrte.tc_latent(phone, m) for m in pros]
        dt = tts.adm.infer_mix([tc] + lats, dw)[..., 0]
        d = dt if forced is None else forced
        tce, totals = ops.length_regulate(tc, d, return_host_totals=True)
        srcs = [ops.maxpool_time(tce, 8)] + [
            ops.maxpool_time(ops.length_regulate(lat, d, l_out=tce.shape[1])[0], 8) for lat in lats]
        step_w = ops.mix_step_weights(pw.to(DEV), d, srcs[0].shape[1])
        codes = tts.plm.infer_mix(srcs, step_w, **SMP)
    assert torch.equal(out["dt"], dt) and out["totals"] == totals
    assert torch.equal(out["prosody_step_weights"], step_w)
    assert torch.equal(step_w.cpu(), torch.from_numpy(MS.step_weights(pw.numpy(), d.cpu().numpy(), srcs[0].shape[1])))
    assert torch.equal(out["p_codes"], codes)
    if len(set(totals)) == 1:
        with torch.no_grad():
            wav = tts.hifi_gan.decode_batch_cl(tts.generator.decode_mel_cl(tce, codes))
        assert torch.equal(out["wav"], wav)
    # the schedule did something: the row mix at each utterance's mean weights decodes other codes
    other = tts.synthesize(phone, melp, forced_durations=forced, prosody_mels=pros, prosody_weights=pw.mean(1),
                           duration_weights=dw, return_intermediates=True, **SMP)
    assert not torch.equal(other["p_codes"], out["p_codes"])


@pytest.mark.parametrize("durations", ["adm", "ragged"])
def test_stream_with_per_phone_weights_equals_synthesize(tts, durations):
    phone, melp, pros, forced = _e2e_inputs(durations)
    pw, dw = _phone_schedules(phone.shape[1])
    kw = dict(forced_durations=forced, prosody_mels=pros, prosody_weights=pw, duration_weights=dw,
              sampling=SMP["sampling"], keys=torch.arange(3, 6))
    ref = tts.synthesize(phone, melp, return_intermediates=True, **kw)
    for cf in (8, max(ref["totals"]) + 100):
        chunks = list(tts.synthesize_stream(phone, melp, chunk_frames=cf, **kw))
        wav = torch.cat([c["wav"] for c in chunks], -1)
        assert torch.equal(chunks[-1]["p_codes"], ref["p_codes"]) and torch.equal(chunks[-1]["dt"], ref["dt"])
        assert wav.shape == ref["wav"].shape
        err = (wav - ref["wav"]).abs().max().item()
        assert err <= 1e-5, (cf, err)


def test_per_phone_rejections(tts):
    phone, melp, pros, forced = _e2e_inputs("equal")
    Tp = phone.shape[1]
    for kw in (dict(prosody_weights=torch.ones(3, Tp + 1, 3)), dict(prosody_weights=torch.ones(3, Tp, 2)),
               dict(prosody_weights=-torch.ones(3, Tp, 3)), dict(duration_weights=torch.zeros(3, Tp, 3)),
               dict(causal_decode=True)):
        args = dict(prosody_mels=pros, prosody_weights=torch.ones(3, Tp, 3))
        args.update(kw)
        with pytest.raises(L.MttsError):
            tts.synthesize(phone, melp, forced_durations=forced, **args)
    with pytest.raises(L.MttsError):
        tts.synthesize_many([(phone[0], melp[0])], prosody_mels=pros, prosody_weights=torch.ones(1, Tp, 3))
