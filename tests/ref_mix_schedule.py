"""numpy / torch CPU restatement of mix schedules (include/megatts2_b200.h, "Prosody and duration schedules"): the phone ->
PLM step rule of mtts_mix_step_weights_f32, and the PLM and ADM mixed decodes with one weight row per step.

Test infrastructure only, built on the per-utterance oracles: each step is tests/ref_prosody_mix.py's pick or
tests/ref_duration_mix.py's readout with that step's row."""
import numpy as np
import torch

import ref_duration_mix as DM
import ref_prosody_mix as PM
from oracle import ref_megatts2 as R


def step_phones(durations, T):
    """durations (B, Tp) int -> (B, T) the phone whose weight row PLM step t takes: the phone owning the most of the mel
    frames [8t, 8t+8) of [0, L_b), the earlier one on a tie; at or past L_b the last phone with a positive duration, or
    phone 0 if none has one.  Negative durations count as 0, as in the length regulator."""
    d = np.maximum(np.asarray(durations, dtype=np.int64), 0)
    B, Tp = d.shape
    out = np.zeros((B, T), dtype=np.int64)
    for b in range(B):
        owner = np.repeat(np.arange(Tp), d[b])                       # frame -> phone
        L = owner.size
        last = int(owner[-1]) if L else 0
        for t in range(T):
            frames = owner[8 * t:min(8 * t + 8, L)]
            if not frames.size:
                out[b, t] = last
                continue
            counts = np.bincount(frames, minlength=Tp)
            out[b, t] = int(np.argmax(counts))                        # argmax takes the first of the largest
    return out


def step_weights(phone_w, durations, T):
    """phone_w (B, Tp, K) -> (B, T, K), the rows of step_phones."""
    pw = np.asarray(phone_w, dtype=np.float32)
    idx = step_phones(durations, T)
    return np.take_along_axis(pw, idx[:, :, None], axis=1)


def plm_infer_mix_steps(sd, tc_latents, cfg, weights, return_logits=False):
    """MegaPLM.infer_mix with a (B, T, K) schedule, greedy: step t's per-source logits from R.plm_step_logits and its pick
    by PM.mix_pick with row (b, t).  -> codes (B, T) [, logits (K, B, T, V), near-tie gaps (B, T)]."""
    K = len(tc_latents)
    B, T, _ = tc_latents[0].shape
    w = np.asarray(weights, dtype=np.float32).reshape(B, T, K)
    codes = torch.full((B, 1), cfg["vq_bins"], dtype=torch.int64)
    all_logits, gaps = [], np.full((B, T), np.inf)
    for t in range(T):
        lg = torch.stack([R.plm_step_logits(sd, tc, codes, cfg) for tc in tc_latents])       # (K, B, V)
        all_logits.append(lg)
        picks = torch.zeros(B, dtype=torch.int64)
        for b in range(B):
            picks[b], gaps[b, t] = PM.mix_pick(lg[:, b].numpy(), w[b, t], t)
        codes = torch.cat([codes, picks[:, None]], 1)
    out = codes[:, 1:]
    return (out, torch.stack(all_logits, 2), gaps) if return_logits else out


def adm_infer_mix_steps(sd, tc_latents, cfg, weights):
    """MegaADM.infer_mix with a (B, T, K) schedule: step t runs DM.adm_step on every source and feeds back
    DM.mix_readout with row (b, t), in the dtype of sd and the latents.  -> (durations (B, T) int32, raw (B, T))."""
    K = len(tc_latents)
    B, T, _ = tc_latents[0].shape
    dtype = tc_latents[0].dtype
    w = np.asarray(weights, dtype=np.float32).reshape(B, T, K)
    p = torch.zeros(B, 1, 1, dtype=dtype)
    for t in range(T):
        ys = torch.stack([DM.adm_step(sd, tc, p, t, cfg)[:, 0, 0] for tc in tc_latents])     # (K, B)
        r = torch.stack([DM.mix_readout(ys[:, b], w[b, t]) for b in range(B)])
        p = torch.cat([p, r.reshape(B, 1, 1)], 1)
    raw = p[:, 1:, 0]
    return (raw + 0.5).to(torch.int32).clamp(1, 128), raw
