"""Host-side pieces of streamed synthesis (Megatts.synthesize_stream): the receptive fields the stream's halos come from,
measured on the CPU oracle, and the chunk schedule (megatts2_b200/stream.py)."""
import pytest
import torch
from hypothesis import given, settings
from hypothesis import strategies as st

import helpers
from megatts2_b200 import stream as SCH
from oracle import ref_megatts2 as R
from oracle import weights


def _reach(out_base, out_pert, f0, frame_of):
    """(lowest, highest) offset from the perturbed input frame f0 of the output frames that changed."""
    d = (out_pert - out_base).abs()
    changed = sorted({frame_of(i) for i in (d > 0).nonzero()[:, -1].tolist()})
    return changed[0] - f0, changed[-1] - f0


def test_decoder_receptive_field_matches_the_oracle(weights_cpu):
    g = helpers.build_g(weights_cpu("g"), "cpu")
    hd = g.decoder.receptive_field()
    assert hd == 20
    sd = R.SD({k: v.double() for k, v in weights_cpu("g").items()}).sub("decoder")
    cfg = weights.G_CFG
    x = torch.randn(1, g.decoder.cfg[0], 64, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    base = R.convnet(sd, x, cfg["dec_kernel"], cfg["dec_n_stack"], cfg["dec_n_block"])
    for f0 in (27, 32):
        x2 = x.clone()
        x2[:, :, f0] += 1.0
        out = R.convnet(sd, x2, cfg["dec_kernel"], cfg["dec_n_stack"], cfg["dec_n_block"])
        lo, hi = _reach(base, out, f0, lambda i: i)
        assert -hd <= lo and hi <= hd and max(-lo, hi) >= hd - 1


def test_vocoder_receptive_field_matches_the_oracle(weights_cpu):
    voc = helpers.build_hifigan(weights_cpu("hifigan"), "cpu").generator
    hv = voc.receptive_field()
    assert 12 <= hv <= 15                       # roughly +-13 frames by hand
    sd = {k: v.double() for k, v in weights_cpu("hifigan").items()}
    pad, hop = weights.HIFIGAN_CFG["inference_padding"], 256
    mel = torch.randn(1, 80, 64, generator=torch.Generator().manual_seed(4), dtype=torch.float64) * 2 - 4
    base = R.hifigan_generator(sd, mel, weights.HIFIGAN_CFG)
    for f0 in (29, 34):
        m2 = mel.clone()
        m2[:, :, f0] += 1.0
        out = R.hifigan_generator(sd, m2, weights.HIFIGAN_CFG)
        lo, hi = _reach(base, out, f0, lambda i: i // hop - pad)
        assert -hv <= lo and hi <= hv and max(-lo, hi) >= hv - 1


@settings(max_examples=400, deadline=None)
@given(L_total=st.integers(1, 700), short=st.integers(0, 700), chunk=st.integers(1, 200), hd=st.integers(0, 40),
       hv=st.integers(5, 30))
def test_chunk_schedule_tiles_the_waveform(L_total, short, chunk, hd, hv):
    pad = 5
    L = max(L_total - short, 0)
    P = SCH.chunk_positions(L_total, chunk, pad)
    assert P[0] == 0 and P[-1] == L_total + 2 * pad and all(x < y for x, y in zip(P, P[1:]))
    plan = SCH.schedule(L, chunk, hd, hv, pad, L_total)
    assert len(plan) == len(P) - 1
    T = -(-L // 8)
    positions, frames, rows, t_prev = [], [], [], 0
    for k, c in enumerate(plan):
        if c is None:
            assert L == 0 or P[k] >= L + 2 * pad
            continue
        assert c.p0 == P[k] and c.p1 == min(P[k + 1], L + 2 * pad)
        positions.append((c.p0, c.p1))
        frames += range(c.a, c.b)
        rows += range(*c.rows)
        va, vb = c.voc
        assert 0 <= va < vb <= L and va % 8 == 0
        # the vocoder window holds every frame the chunk's samples read; an inner edge keeps a full halo
        assert va == 0 or c.p0 - pad - va >= hv
        assert vb == L or vb - (c.p1 - pad) >= hv
        assert set(range(va, vb)) <= set(rows)
        if c.dec is not None:
            da, db = c.dec
            assert 0 <= da < db <= L and da % 8 == 0
            assert da == 0 or c.rows[0] - da >= hd
            assert db == L or db - c.rows[1] >= hd
            assert (db - 1) // 8 < c.t1                 # the decoder window's last code is decoded
        assert t_prev <= c.t1 <= T
        t_prev = c.t1
    if L > 0:
        # the chunks tile the utterance's positions [0, L + 2 pad) and its frames [0, L) exactly once
        assert positions[0][0] == 0 and positions[-1][1] == L + 2 * pad
        assert all(x[1] == y[0] for x, y in zip(positions, positions[1:]))
        assert frames == list(range(L))
        assert rows == list(range(L))                    # every mel row is decoded once


def test_chunk_schedule_single_chunk_and_errors():
    (c,) = SCH.schedule(40, 64, 20, 14, 5)
    assert (c.p0, c.p1, c.a, c.b, c.rows, c.dec, c.voc, c.t1) == (0, 50, 0, 40, (0, 40), (0, 40), (0, 40), 5)
    with pytest.raises(ValueError):
        SCH.chunk_positions(0, 8, 5)
    with pytest.raises(ValueError):
        SCH.schedule(9, 8, 20, 14, 5, L_total=8)
