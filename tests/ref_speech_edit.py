"""Restatements of speech editing (megatts2_b200/edit.py, MegaPLM.infer(pinned=)) for the tests.

Test infrastructure only.  ``code_pins`` restates the pin rule frame by frame: each frame of the edited utterance is
classed as a prefix, new or suffix frame, a suffix frame is traced back to its original frame, and the original block a
block keeps is chosen by explicit counts.  ``plm_infer_pinned`` is the fp64 PLM decode with the pins teacher-forced,
built on tests/ref_plm_context.py's step."""
from collections import Counter

import torch

import ref_plm_context as RC
from oracle import ref_sampling as RS


def code_pins(orig_durations, orig_codes, span, n_new, new_frames, T):
    """(B, T) int pins from the original durations (B, Tp_o), codes (B, T_o), span (B, 2), the new phones' counts n
    and their frame counts L_n per row."""
    B = len(orig_durations)
    out = torch.full((B, T), -1, dtype=torch.int64)
    for r in range(B):
        d = [int(x) for x in orig_durations[r]]
        a, b = int(span[r][0]), int(span[r][1])
        F_a, L_o, F_s, L_n = sum(d[:a]), sum(d[a:b]), sum(d[b:]), int(new_frames[r])
        N_e = F_a + L_n + F_s
        for k in range(T):
            frames = [f for f in range(8 * k, 8 * k + 8) if f < N_e]
            if not frames:
                out[r, k] = 0
                continue
            kinds = ["p" if f < F_a else "n" if f < F_a + L_n else "s" for f in frames]
            if kinds == ["p"] * 8:
                out[r, k] = int(orig_codes[r][k])
            elif set(kinds) == {"s"}:
                # the i-th suffix frame, f = F_a + L_n + i, is the original frame F_a + L_o + i
                src = Counter((F_a + L_o + (f - F_a - L_n)) // 8 for f in frames)
                best = max(src.values())
                out[r, k] = int(orig_codes[r][min(q for q, c in src.items() if c == best)])
    return out


def plm_infer_pinned(sd, tc, cfg, pins, ctx_tc=None, ctx_codes=None, sampling=None, keys=None):
    """The PLM decode (non-causal, as MegaPLM.infer) with pins[b, j] >= 0 written into the history in place of the pick,
    in the dtype of ``sd`` and ``tc``.  -> codes (B, T), logits (B, T, V): every step's logits, pinned ones included."""
    B, T, _ = tc.shape
    if ctx_tc is None:
        ctx_tc, ctx_codes = tc.new_zeros(1, 0, tc.shape[2]), torch.zeros(1, 0, dtype=torch.int64)
    lat, codes = RC.concat(ctx_tc, ctx_codes, tc, cfg["vq_bins"])
    keys = list(range(B)) if keys is None else [int(k) for k in keys]
    logits = []
    for j in range(T):
        lg = RC.step_logits(sd, lat, codes, cfg, False)
        logits.append(lg)
        if sampling is None:
            pick = lg.argmax(-1)
        else:
            t, k, p, seed = sampling
            pick = torch.tensor([RS.sample_row(lg[b].float().numpy(), j, t, k, p, seed, keys[b])[0] for b in range(B)])
        pick = torch.where(pins[:, j] >= 0, pins[:, j].to(torch.int64), pick)
        codes = torch.cat([codes, pick.reshape(B, 1)], 1)
    return codes[:, codes.shape[1] - T:], torch.stack(logits, 1)
