"""GPU: speech editing (include/megatts2_b200.h, code pins; megatts2_b200/edit.py).  MegaPLM.infer(pinned=) against
the unpinned decode and the fp64 restatement with the pins teacher-forced (tests/ref_speech_edit.py), the exactness of
skipped steps, sampling and replay, the C entry's free pin values, and Megatts.edit end to end.

Bars: free steps' logits within the PLM tests' 2e-3 of the restatement evaluated on the device's own code prefix, and
greedy picks equal its argmax except on rows whose two best fp32 logits are within NEAR (relative, floor 1); every
identity bit for bit."""
import ctypes as C

import pytest
import torch

import helpers
import ref_plm_context as PC
import ref_speech_edit as RE
from megatts2_b200 import _lib as L
from megatts2_b200 import graphs, ops, pack
from megatts2_b200.models.megatts2 import PLMContext
from megatts2_b200.sampling import Sampling
from oracle import ref_megatts2 as R
from oracle import weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = "cuda"
CFG = weights.PLM_CFG
V = CFG["vq_bins"]
NEAR = 1e-5
TOL = 2e-3
ENGINES = pytest.mark.parametrize("engine", [pack.ENGINE_F16X2, pack.ENGINE_BF16X3, pack.ENGINE_FFMA],
                                  ids=["f16x2", "bf16x3", "ffma"])
SMP = Sampling(temperature=0.9, top_k=40, seed=5)


def gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def tts(weights_cpu):
    return helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)


def latent(B, T, seed):
    return torch.randn(B, T, 512, generator=gen(seed)).abs()


def ctx_of(seed, Bc=1, P=5):
    return PLMContext(torch.randn(Bc, P, 512, generator=gen(seed)).abs().to(DEV),
                      torch.randint(0, V, (Bc, P), generator=gen(seed + 1)).to(DEV))


def pins_of(B, T, seed, frac=0.4):
    g = gen(seed)
    p = torch.randint(0, V, (B, T), generator=g)
    return torch.where(torch.rand(B, T, generator=g) < frac, p, torch.full_like(p, -1)).to(torch.int32)


def near_tie(row):
    top2 = torch.topk(row.double(), 2).values
    return (top2[0] - top2[1]).item() / max(1.0, abs(top2[0].item())) <= NEAR


# ------------------------------------------------------------------------------ identities of the pinned decode
@ENGINES
def test_all_free_pins_equal_the_unpinned_decode(tts, engine):
    plm = tts.plm
    B, T = 3, 12
    tc = latent(B, T, 1).to(DEV)
    free = torch.full((B, T), -1, dtype=torch.int32)
    with pack.engine_scope(engine):
        for kw in (dict(), dict(sampling=SMP, keys=[4, 5, 6]), dict(context=ctx_of(2))):
            for _ in range(3):                                  # eager, capture, replay
                a = plm.infer(tc, return_logits=True, **kw)
                b = plm.infer(tc, return_logits=True, pinned=free, **kw)
                c = plm.infer(tc, pinned=free, **kw)
                assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[0], c), kw


@ENGINES
def test_pinned_decode_against_the_fp64_restatement(weights_cpu, tts, engine):
    sd = PC.sd_as(weights_cpu("plm"), torch.float64)
    B, T = 3, 10
    tc = latent(B, T, 10)
    pins = pins_of(B, T, 11)
    pins[:, 4] = torch.tensor([7, 8, 9], dtype=torch.int32)      # a step pinned in every row
    with pack.engine_scope(engine):
        codes, logits = tts.plm.infer(tc.to(DEV), return_logits=True, pinned=pins)
    codes, logits = codes.cpu(), logits.cpu()
    on = pins >= 0
    assert torch.equal(codes[on], pins[on].long())
    hist = torch.cat([torch.full((B, 1), V, dtype=torch.int64), codes], 1)
    worst, ties = 0.0, 0
    for j in range(T):
        ref = R.plm_step_logits(R.SD(sd), tc.double(), hist[:, :j + 1], CFG)   # the device's own prefix, pins included
        err = (logits[:, j].double() - ref).abs().max().item()
        worst = max(worst, err)
        assert err <= TOL, (j, err)
        for b in range(B):
            if not on[b, j] and int(codes[b, j]) != int(ref[b].argmax()):
                assert near_tie(ref[b]), (j, b)
                ties += 1
    # the restatement's own decode with the pins teacher-forced agrees where no near-tie intervened
    want, _ = RE.plm_infer_pinned(sd, tc.double(), CFG, pins)
    if ties == 0:
        assert torch.equal(codes, want)
    print(f"{engine}: max |logits - restatement| = {worst:.3g}, {ties} near-tie picks")
    helpers.record("speech_edit_pinned_logits", dict(engine=engine, max_abs=worst, ties=ties))


@ENGINES
def test_pinning_a_prefix_to_infers_codes_reproduces_infer(tts, engine):
    plm = tts.plm
    B, T = 3, 14
    tc = latent(B, T, 20).to(DEV)
    with pack.engine_scope(engine):
        for kw in (dict(), dict(sampling=SMP, keys=[1, 2, 3]), dict(context=ctx_of(21, Bc=3))):
            ref = plm.infer(tc, **kw)
            for j in (1, 5, T - 1, T):
                pins = torch.full((B, T), -1, dtype=torch.int32)
                pins[:, :j] = ref[:, :j].cpu().to(torch.int32)
                for _ in range(3):
                    assert torch.equal(plm.infer(tc, pinned=pins, **kw), ref), (kw, j)


@ENGINES
def test_skipping_interior_runs_equals_running_every_step(tts, engine):
    plm = tts.plm
    B, T = 4, 16
    tc = latent(B, T, 30).to(DEV)
    pins = pins_of(B, T, 31, frac=0.5)
    pins[:, 3:6] = torch.randint(0, V, (B, 3), generator=gen(32)).to(torch.int32)
    pins[:, 10] = 5
    with pack.engine_scope(engine):
        for kw in (dict(), dict(sampling=SMP, keys=[9, 8, 7, 6]), dict(context=ctx_of(33))):
            full = plm.infer(tc, return_logits=True, pinned=pins, **kw)[0]
            for _ in range(3):
                assert torch.equal(plm.infer(tc, pinned=pins, **kw), full), kw


def test_a_pin_leaves_other_rows_draws_unchanged(tts):
    plm = tts.plm
    B, T = 4, 12
    tc = latent(B, T, 40).to(DEV)
    keys = [11, 12, 13, 14]
    ref = plm.infer(tc, sampling=SMP, keys=keys)
    pins = torch.full((B, T), -1, dtype=torch.int32)
    pins[2] = (ref[2].cpu() + 1).remainder(V).to(torch.int32)       # row 2 pinned everywhere to other codes
    got = plm.infer(tc, sampling=SMP, keys=keys, pinned=pins)
    assert torch.equal(got[2].cpu(), pins[2].long())
    assert torch.equal(got[[0, 1, 3]], ref[[0, 1, 3]])


def test_new_pin_values_replay_without_a_capture(tts):
    plm = tts.plm
    B, T = 3, 10
    tc = latent(B, T, 50).to(DEV)
    mask = pins_of(B, T, 51) >= 0

    def pins(seed):
        return torch.where(mask, torch.randint(0, V, (B, T), generator=gen(seed)), -1).to(torch.int32)
    for _ in range(2):                                                  # warm-up, capture
        plm.infer(tc, pinned=pins(52))
    cache = plm._graphs("pinned").cache
    n_graphs, n_replayed = len(cache), graphs.replayed_launches
    outs = set()
    for seed in range(53, 57):
        got = plm.infer(tc, pinned=pins(seed))
        with graphs.disabled():
            want = plm.infer(tc, pinned=pins(seed))
        assert torch.equal(got, want), seed
        assert torch.equal(got.cpu()[mask], pins(seed)[mask].long())
        outs.add(tuple(got.flatten().tolist()))
    assert len(cache) == n_graphs and graphs.replayed_launches > n_replayed
    assert len(outs) == 4


def test_out_of_range_pins_at_the_c_entry_are_free(tts):
    """V, V + 1 and -5 passed straight to mtts_plm_infer_pinned_f32 leave the step free: the decode equals infer's."""
    plm = tts.plm
    B, T = 3, 8
    tc = latent(B, T, 60).to(DEV)
    with graphs.disabled():
        ref_codes, ref_logits = plm.infer(tc, return_logits=True)
    pins = torch.tensor([V, V + 1, -5], dtype=torch.int32).repeat_interleave(T).reshape(B, T).contiguous().to(DEV)
    lib = L.lib()
    pl = plm._plan_get(tc.device, T)
    m = C.byref(pl.struct)
    state = torch.full((B, T + 1), V, dtype=torch.int64, device=DEV)
    codes = torch.zeros(B, T, dtype=torch.int64, device=DEV)
    logits = torch.zeros(B, T, V, device=DEV)
    ws = ops.workspace(lib.mtts_plm_infer_ctx_workspace_bytes(m, B, 0, T), tc.device)
    L.check(lib.mtts_plm_infer_pinned_f32(m, tc.data_ptr(), tc.stride(0), tc.stride(1), B, T, None, 0, 0, None, 0, 0, 0,
                                          T, state.data_ptr(), codes.data_ptr(), logits.data_ptr(), None,
                                          pins.data_ptr(), T, ws.data_ptr(), ws.numel(), ops._stream()))
    assert torch.equal(codes, ref_codes) and torch.equal(state[:, 1:], ref_codes) and torch.equal(logits, ref_logits)


# ------------------------------------------------------------------------------ Megatts.edit
def _original(tts, B=3, Tp=9, seed=70, **kw):
    phone = torch.randint(0, 320, (B, Tp), generator=gen(seed)).to(DEV)
    melp = (torch.randn(B, 56, 80, generator=gen(seed + 1)) * 2 - 4).to(DEV)
    d = torch.randint(2, 12, (B, Tp), generator=gen(seed + 2), dtype=torch.int32).to(DEV)
    out = tts.synthesize(phone, melp, forced_durations=d, return_intermediates=True, **kw)
    return phone, melp, d, out


def _replace(phone, span, new):
    """Edited phone rows: row r's span [a, b) replaced by new[r] (all rows the same length)."""
    rows = [torch.cat([phone[r, :a], torch.tensor(new[r], device=DEV), phone[r, b:]]) for r, (a, b) in enumerate(span)]
    return torch.stack(rows)


def test_identity_edit_returns_the_original(tts):
    phone, melp, d, out = _original(tts)
    n0 = ops.launch_count()
    tts.plm.infer(out["tc8"], pinned=out["p_codes"].cpu().to(torch.int32))   # every step pinned: nothing enqueued
    assert ops.launch_count() == n0
    span = torch.zeros(3, 2, dtype=torch.int64)
    got = tts.edit(phone, melp, phone, d, out["p_codes"], span, return_intermediates=True)
    assert (got["code_pins"] >= 0).all()
    assert torch.equal(got["dt"], d)
    for r, n in enumerate(out["totals"]):          # a step past a row's end, which no one reads, is pinned to 0
        k = -(-n // 8)
        assert torch.equal(got["p_codes"][r, :k], out["p_codes"][r, :k]) and (got["p_codes"][r, k:] == 0).all()
    assert torch.equal(got["wav"], out["wav"]) and got["wav_lens"] == out["wav_lens"]
    assert got["edit_frames"].tolist() == [[0, 0]] * 3


def test_word_replacement_equals_the_composed_pieces(tts):
    phone, melp, d, orig = _original(tts, seed=80)
    span = [(2, 4), (3, 4), (5, 7)]
    new = [[301, 302, 303], [304, 305], [306, 307, 308]]            # one phone more in every row
    ph_e = _replace(phone, span, new)
    sf = [9, 14, 7]
    got = tts.edit(ph_e, melp, phone, d, orig["p_codes"], torch.tensor(span), span_frames=sf,
                   return_intermediates=True)
    # the pieces: MRTE, the ADM with pins and the fit, length regulation, the pin gather, infer(pinned=), decoder, vocoder
    B, Tp_e = ph_e.shape
    dc = d.cpu()
    pins = torch.full((B, Tp_e), -1, dtype=torch.int32)
    for r, (a, b) in enumerate(span):
        n = len(new[r])
        pins[r, :a], pins[r, a + n:] = dc[r, :a], dc[r, b:]
    total = [int(dc[r, :a].sum()) + sf[r] + int(dc[r, b:].sum()) for r, (a, b) in enumerate(span)]
    tc_latent = tts.generator.mrte.tc_latent(ph_e, melp)
    _, raw = tts.adm.infer(tc_latent, return_raw=True, pinned=pins)
    dt = ops.fit_durations(raw, None, torch.tensor(total, dtype=torch.int32), pins)
    assert torch.equal(got["dt"], dt)
    assert dt.sum(1).tolist() == total
    tc_expand, totals = ops.length_regulate(tc_latent, dt, return_host_totals=True)
    tc8 = ops.maxpool_time(tc_expand, 8)
    T = tc8.shape[1]
    L_n = [totals[r] - int(dc[r, :a].sum()) - int(dc[r, b:].sum()) for r, (a, b) in enumerate(span)]
    cp = RE.code_pins(dc.tolist(), orig["p_codes"].cpu().tolist(), span, [len(x) for x in new], L_n, T)
    assert torch.equal(got["code_pins"].long(), cp)
    p_codes = tts.plm.infer(tc8, pinned=cp)
    assert torch.equal(got["p_codes"], p_codes)
    on = cp >= 0
    assert torch.equal(p_codes.cpu()[on], cp[on])
    assert (~on).any() and on.any()
    wav = torch.zeros_like(got["wav"])
    for Lg in sorted(set(totals)):
        idx = [r for r in range(B) if totals[r] == Lg]
        mel = tts.generator.decode_mel_cl(tc_expand[idx, :Lg].contiguous(), p_codes[idx, :(Lg + 7) // 8].contiguous())
        w = tts.hifi_gan.decode_batch_cl(mel)
        wav[idx, :, :w.shape[-1]] = w
    assert torch.equal(got["wav"], wav)
    F_a = [int(dc[r, :a].sum()) for r, (a, _) in enumerate(span)]
    assert got["edit_frames"].tolist() == [[F_a[r], F_a[r] + sf[r]] for r in range(B)]


def test_span_frames_equal_to_the_replaced_frames_keep_the_prefix_and_suffix_codes(tts):
    phone, melp, d, orig = _original(tts, seed=90)
    span = [(3, 5), (1, 3), (4, 6)]
    new = [[311, 312], [313, 314], [315, 316]]
    dc = d.cpu()
    L_o = [int(dc[r, a:b].sum()) for r, (a, b) in enumerate(span)]
    got = tts.edit(_replace(phone, span, new), melp, phone, d, orig["p_codes"], torch.tensor(span), span_frames=L_o,
                   return_intermediates=True)
    assert got["totals"] == orig["totals"]
    for r, (a, b) in enumerate(span):
        F_a, end = int(dc[r, :a].sum()), int(dc[r, :b].sum())
        for k in range(got["p_codes"].shape[1]):
            if 8 * k + 8 <= F_a or (8 * k >= end and 8 * k < orig["totals"][r]):
                assert int(got["p_codes"][r, k]) == int(orig["p_codes"][r, k]), (r, k)
        assert torch.equal(got["dt"][r, :a].cpu(), dc[r, :a]) and torch.equal(got["dt"][r, a + 2:].cpu(), dc[r, b:])


def test_sampled_takes_differ_only_at_free_steps(tts):
    phone, melp, d, orig = _original(tts, seed=100)
    span = [(2, 3), (4, 5), (6, 7)]
    new = [[317, 300], [301, 302], [303, 304]]
    ph_e = _replace(phone, span, new)
    takes = [tts.edit(ph_e, melp, phone, d, orig["p_codes"], torch.tensor(span), span_frames=[12, 12, 12],
                      sampling=SMP, keys=[k, k + 1, k + 2], return_intermediates=True) for k in (0, 100)]
    on = takes[0]["code_pins"] >= 0
    assert torch.equal(takes[0]["code_pins"], takes[1]["code_pins"])
    a, b = takes[0]["p_codes"].cpu(), takes[1]["p_codes"].cpu()
    assert torch.equal(a[on], b[on]) and torch.equal(a[on], takes[0]["code_pins"][on].long())
    assert not torch.equal(a[~on], b[~on])
    assert torch.equal(takes[0]["dt"], takes[1]["dt"])
