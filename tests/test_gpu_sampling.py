"""GPU: the opt-in PLM sampler (csrc/sample.cu) against its numpy oracle (oracle/ref_sampling.py), and the sampled decode
through MegaPLM.infer / infer_causal and Megatts.synthesize.

Bars: Philox words and the support of the filters exact; picks equal the oracle's except on rows whose two best fp64
scores are within 1e-5 (relative, floor 1) - fp32 scores against fp64 ones; the distribution of 2^20 draws passes a
chi-square test against the fp64 target at p >= 1e-6; the greedy limits bit-identical to the greedy decode."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers
from oracle import ref_megatts2 as R
from oracle import ref_sampling as RS
from oracle import weights

pytestmark = pytest.mark.gpu
DEV = "cuda"
NEAR = 1e-5


def gen(seed):
    return torch.Generator().manual_seed(seed)


def maxerr(a, b):
    return (a.detach().float().cpu() - b.detach().float().cpu()).abs().max().item()


def S(**kw):
    from megatts2_b200.sampling import Sampling
    return Sampling(**kw)


def draw(z, step, s, keys):
    from megatts2_b200 import ops
    return ops.sample_rows(z if z.is_cuda else z.to(DEV), step, s, torch.as_tensor(keys).to(DEV)).cpu().numpy()


@pytest.fixture(scope="module")
def PLM(weights_cpu):
    return helpers.build_plm(weights_cpu("plm"), DEV)


# ------------------------------------------------------------------------------ kernel level
def test_device_philox_words_equal_the_oracle():
    from megatts2_b200 import ops
    rng = np.random.default_rng(3)
    n = 1 << 14
    ctr = rng.integers(0, 2 ** 32, (n, 4), dtype=np.uint64)
    key = rng.integers(0, 2 ** 32, (n, 2), dtype=np.uint64)
    ctr[:3] = [[0] * 4, [0xffffffff] * 4, [0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344]]
    key[:3] = [[0, 0], [0xffffffff] * 2, [0xa4093822, 0x299f31d0]]
    got = ops.philox4x32_10(torch.from_numpy(ctr.astype(np.int64)).to(DEV), torch.from_numpy(key.astype(np.int64)).to(DEV))
    got = got.cpu().numpy().astype(np.uint64)
    assert np.array_equal(got, RS.philox4x32_10(ctr, key).astype(np.uint64))
    assert [int(w) for w in got[0]] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    # the sampler's layout: token i of step t under (seed, key) reads word i & 3 of counter (i >> 2, t, key_lo, key_hi)
    for seed, kk, t in ((0, 0, 0), (2 ** 64 - 1, 2 ** 63 + 12345, 511), (int(rng.integers(2 ** 63)), int(rng.integers(2 ** 63)), 77)):
        i = np.arange(1024, dtype=np.uint64)
        c = np.stack([i >> np.uint64(2), np.full_like(i, t), np.full_like(i, kk & 0xFFFFFFFF), np.full_like(i, kk >> 32)], -1)
        k = np.tile(np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64), (1024, 1))
        dev = ops.philox4x32_10(torch.from_numpy(c.astype(np.int64)).to(DEV), torch.from_numpy(k.astype(np.int64)).to(DEV))
        dev = dev.cpu().numpy()[np.arange(1024), (i & np.uint64(3)).astype(np.int64)]
        assert np.array_equal(dev.astype(np.uint64), RS.words(seed, kk, t, i).astype(np.uint64))


COMBOS = [dict(temperature=1.0), dict(temperature=0.7, top_k=20), dict(top_p=0.9),
          dict(temperature=1.3, top_k=50, top_p=0.8), dict(temperature=0.5, top_k=5000), dict(temperature=2.0, top_p=0.999),
          dict(temperature=1.0, top_k=2)]


@pytest.mark.parametrize("V", [1024, 1000, 37])
@pytest.mark.parametrize("ci", range(len(COMBOS)))
def test_picks_agree_with_the_oracle(ci, V):
    kw = COMBOS[ci]
    rows, step = 256, 5 + ci
    z = torch.randn(rows, V, generator=gen(100 * ci + V)) * 3
    keys = torch.randint(0, 2 ** 62, (rows,), generator=gen(7 + ci))
    s = S(seed=2 ** 64 - 1 - 1000 * ci - V, **kw)
    got = draw(z, step, s, keys)
    want, gaps = RS.sample_rows(z.numpy(), step, s.temperature, s.top_k, s.top_p, s.seed, keys.numpy())
    bad = got != want
    print(f"{kw} V={V}: {int(bad.sum())} of {rows} picks differ from the oracle")
    assert (gaps[bad] <= NEAR).all(), (np.nonzero(bad)[0], gaps[bad])
    assert bad.sum() <= 2


@pytest.mark.parametrize("ci", [1, 2, 3, 6])
def test_no_draw_outside_the_kept_set(ci):
    kw = COMBOS[ci]
    V, n = 1024, 1 << 16
    z = torch.randn(V, generator=gen(31 + ci)) * 2
    s = S(seed=99 + ci, **kw)
    got = draw(z.to(DEV).expand(n, V), 3, s, torch.arange(n))
    kept, _ = RS.kept_set(RS.tempered(z.numpy(), s.temperature), s.top_k, s.top_p)
    assert set(np.unique(got).tolist()) <= set(kept.tolist())
    # and on random rows, each against its own kept set
    zr = torch.randn(512, V, generator=gen(41 + ci)) * 3
    got = draw(zr, 9, s, torch.arange(512) * 3)
    for r in range(512):
        kept, _ = RS.kept_set(RS.tempered(zr[r].numpy(), s.temperature), s.top_k, s.top_p)
        assert got[r] in set(kept.tolist())


@pytest.mark.parametrize("kw", [dict(temperature=1.0), dict(temperature=0.7, top_k=20), dict(top_p=0.9)])
def test_distribution_of_two_to_the_twenty_draws(kw):
    from scipy import stats
    V, n = 1024, 1 << 20
    z = torch.randn(V, generator=gen(5)) * 2
    s = S(seed=2024, **kw)
    got = draw(z.to(DEV).expand(n, V), 17, s, torch.arange(n))
    obs = np.bincount(got, minlength=V).astype(np.float64)
    p = RS.target_distribution(z.numpy(), s.temperature, s.top_k, s.top_p)
    assert obs[p == 0].sum() == 0
    exp = n * p
    big = exp >= 5
    o = np.append(obs[big], obs[~big].sum())
    e = np.append(exp[big], exp[~big].sum())
    if e[-1] == 0:
        o, e = o[:-1], e[:-1]
    res = stats.chisquare(o, e * (o.sum() / e.sum()))
    print(f"{kw}: chi2 {res.statistic:.1f} over {len(o) - 1} dof, p-value {res.pvalue:.3g}")
    assert res.pvalue >= 1e-6


@pytest.mark.parametrize("ci", [0, 3])
def test_pick_does_not_depend_on_position_or_batch(ci):
    s = S(seed=77, **COMBOS[ci])
    z = torch.randn(64, 1024, generator=gen(61)) * 3
    keys = torch.randint(0, 2 ** 62, (64,), generator=gen(62))
    full = draw(z, 4, s, keys)
    perm = torch.randperm(64, generator=gen(63))
    assert np.array_equal(draw(z[perm], 4, s, keys[perm]), full[perm.numpy()])
    for a, b in ((5, 6), (10, 40), (0, 64)):
        assert np.array_equal(draw(z[a:b], 4, s, keys[a:b]), full[a:b])
    assert np.array_equal(draw(z[7].expand(3, 1024), 4, s, keys[7].repeat(3)), np.repeat(full[7], 3))


def test_edge_rows():
    V = 64
    rows = []
    z = torch.randn(V, generator=gen(71)).numpy().astype(np.float32)
    r = z.copy(); r[:4] = np.nan; rows.append(r)                                    # NaN is never a candidate
    r = z.copy(); r[7] = np.inf; r[3] = np.inf; rows.append(r)                      # lowest +inf index: 3
    rows.append(np.full(V, -np.inf, np.float32))                                    # no finite value: 0
    rows.append(np.full(V, np.nan, np.float32))
    r = np.full(V, np.nan, np.float32); r[::2] = -np.inf; rows.append(r)
    rows.append(np.zeros(V, np.float32))                                            # all equal
    r = z.copy(); r[::3] = -np.inf; rows.append(r)
    r = np.full(V, np.nan, np.float32); r[9] = -5.0; rows.append(r)                 # one candidate
    r = z.copy(); r[20] = 2e38; r[11] = 3e38; rows.append(r)                        # +inf (both) at temperature 0.5
    r = z.copy(); r[30] = -0.0; r[31] = 0.0; rows.append(r)
    zz = torch.from_numpy(np.stack(rows))
    keys = np.arange(len(rows)) + 1000
    for kw in COMBOS + [dict(temperature=0.0), dict(top_k=1), dict(temperature=0.5), dict(temperature=0.5, top_k=3)]:
        s = S(seed=5, **kw)
        got = draw(zz, 2, s, keys)
        want, _ = RS.sample_rows(zz.numpy(), 2, s.temperature, s.top_k, s.top_p, s.seed, keys)
        assert np.array_equal(got, want), (kw, got, want)
        assert got[0] >= 4 and got[1] == 3 and got[2] == 0 and got[3] == 0 and got[4] == 0 and got[6] % 3 != 0
        assert got[7] == 9
        if s.temperature == 0.5 and s.top_k != 1:
            assert got[8] == 11
    for kw, allowed in ((dict(top_k=3), {0, 1, 2}), (dict(top_p=0.5), set(range(32)))):
        got = draw(torch.zeros(V, device=DEV).expand(4096, V), 0, S(seed=8, **kw), torch.arange(4096))
        assert set(np.unique(got).tolist()) == allowed


# ------------------------------------------------------------------------------ model level
def test_greedy_limits_are_bit_identical(golden, PLM):
    tc = golden("plm")["tc8"].to(DEV)
    ids, lg = PLM.infer(tc, return_logits=True)
    cids, clg = PLM.infer_causal(tc, return_logits=True)
    for s in (S(top_k=1, seed=3), S(temperature=0.0, seed=3), S(top_p=1e-9, seed=3)):
        for _ in range(3):                    # eager, capture + replay, replay
            i2, l2 = PLM.infer(tc, return_logits=True, sampling=s)
            assert torch.equal(i2, ids) and torch.equal(l2, lg), s
        i2, l2 = PLM.infer_causal(tc, return_logits=True, sampling=s)
        assert torch.equal(i2, cids) and torch.equal(l2, clg), s


@pytest.mark.parametrize("kw", [dict(temperature=1.0), dict(temperature=1.2, top_k=50, top_p=0.9)])
def test_sampled_decode_matches_the_oracle(golden, weights_cpu, PLM, kw):
    tc = golden("plm")["tc8"]
    B, T = tc.shape[:2]
    keys = [3, 2 ** 40 + 1]
    s = S(seed=11, **kw)
    sd = R.SD(weights_cpu("plm"))
    for decode in (PLM.infer, PLM.infer_causal):
        ids, lg = decode(tc.to(DEV), return_logits=True, sampling=s, keys=keys)
        ids, lg = ids.cpu(), lg.cpu()
        n_bad = 0
        for t in range(T):
            want, gaps = RS.sample_rows(lg[:, t].numpy(), t, s.temperature, s.top_k, s.top_p, s.seed, keys)
            bad = ids[:, t].numpy() != want
            assert (gaps[bad] <= NEAR).all()
            n_bad += int(bad.sum())
        assert n_bad <= 1
        codes_in = torch.cat([torch.full((B, 1), 1024), ids], 1)
        if decode == PLM.infer:
            # the oracle's non-causal step on the sampled prefix reproduces every step's logits
            for t in range(T):
                assert maxerr(lg[:, t], R.plm_step_logits(sd, tc, codes_in[:, :t + 1], weights.PLM_CFG)) < 2e-3
        else:
            fwd, _ = PLM(tc.to(DEV), codes_in.to(DEV), torch.full((B,), T, dtype=torch.int32, device=DEV))
            assert maxerr(fwd, lg) < 2e-3
    # the full oracle decode (its own logits, its own draws) agrees wherever no step was a near-tie
    ref_ids = RS.plm_infer_sampled(sd, tc, weights.PLM_CFG, s.temperature, s.top_k, s.top_p, s.seed, keys)
    ids = PLM.infer(tc.to(DEV), sampling=s, keys=keys).cpu()
    print(f"{kw}: device ids equal the oracle decode on {float((ids == ref_ids).float().mean()):.3f} of the positions")


def test_seed_and_keys_are_graph_inputs(PLM):
    from megatts2_b200 import graphs
    tc = F.relu(torch.randn(4, 12, 512, generator=gen(81))).to(DEV)
    s1, s2 = S(temperature=1.5, seed=1), S(temperature=1.5, seed=2)
    PLM._graphs().clear()
    outs = [PLM.infer(tc, sampling=s1) for _ in range(3)]          # eager, capture + replay, replay
    assert all(torch.equal(o, outs[0]) for o in outs)
    if graphs.enabled():
        assert any(len(e) == 4 for e in PLM._graphs().cache.values())
    r2 = PLM.infer(tc, sampling=s2)                                  # replay, new seed
    r3 = PLM.infer(tc, sampling=s1, keys=[9, 8, 7, 6])               # replay, new keys
    with graphs.disabled():
        e1, e2 = PLM.infer(tc, sampling=s1), PLM.infer(tc, sampling=s2)
        e3 = PLM.infer(tc, sampling=s1, keys=[9, 8, 7, 6])
    assert torch.equal(e1, outs[0]) and torch.equal(r2, e2) and torch.equal(r3, e3)
    assert not torch.equal(r2, outs[0]) and not torch.equal(r3, outs[0])
    assert torch.equal(PLM.infer(tc), PLM.infer(tc, sampling=S(temperature=0.0, seed=1)))


def test_keys_select_the_take(PLM):
    s = S(temperature=1.5, seed=5)
    one = F.relu(torch.randn(1, 16, 512, generator=gen(91))).to(DEV)
    two = one.expand(2, 16, 512).contiguous()
    a = PLM.infer(two, sampling=s, keys=[7, 7])
    b = PLM.infer(two, sampling=s, keys=[7, 8])
    assert torch.equal(a[0], a[1]) and torch.equal(b[0], a[0]) and not torch.equal(b[0], b[1])
    assert torch.equal(PLM.infer(one, sampling=s, keys=[7])[0], a[0])
    four = F.relu(torch.randn(4, 16, 512, generator=gen(92))).to(DEV)
    full = PLM.infer(four, sampling=s, keys=[10, 11, 12, 13])
    assert torch.equal(PLM.infer(four[2:3], sampling=s, keys=[12])[0], full[2])
    assert torch.equal(PLM.infer_causal(four, sampling=s, keys=[10, 11, 12, 13])[2],
                       PLM.infer_causal(four[2:3], sampling=s, keys=[12])[0])


def test_synthesize_with_sampling(golden, weights_cpu):
    g = golden("e2e")
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    s = S(temperature=1.0, top_p=0.95, seed=21)
    args = (g["phone"].to(DEV), g["mel_prompt"].to(DEV))
    o = tts.synthesize(*args, forced_durations=g["dt_used"].to(DEV), return_intermediates=True, sampling=s)
    assert torch.equal(o["p_codes"], tts.plm.infer(o["tc8"], sampling=s))
    greedy = tts.synthesize(*args, forced_durations=g["dt_used"].to(DEV), return_intermediates=True)
    assert torch.equal(greedy["p_codes"].cpu(), g["p_codes"]) and torch.equal(o["dt"], greedy["dt"])
    o2 = tts.synthesize(*args, forced_durations=g["dt_used"].to(DEV), return_intermediates=True, sampling=s, keys=[5])
    assert torch.equal(o2["p_codes"], tts.plm.infer(o2["tc8"], sampling=s, keys=[5]))
    # synthesize_many keys utterance i by its index: the batching does not change what it draws
    phone = torch.randint(0, 320, (2, 6), generator=gen(44)).to(DEV)
    melp = (torch.randn(2, 48, 80, generator=gen(45)) * 2 - 4).to(DEV)
    p2 = torch.randint(0, 320, (4,), generator=gen(46)).to(DEV)
    m2 = (torch.randn(40, 80, generator=gen(47)) * 2 - 4).to(DEV)
    items = [(phone[0], melp[0]), (p2, m2), (phone[1], melp[1])]
    wide = tts.synthesize_many(items, max_batch=64, sampling=s)
    narrow = tts.synthesize_many(items, max_batch=1, sampling=s)
    assert all(torch.equal(a, b) for a, b in zip(wide, narrow))
    w2, n2 = tts.synthesize(phone[1:2], melp[1:2], return_lengths=True, sampling=s, keys=[2])
    assert torch.equal(wide[2], w2[0, 0, :n2[0]])
