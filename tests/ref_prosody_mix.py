"""numpy / fp64 restatement of the prosody mix (include/megatts2_b200.h, mtts_mix_logprob_rows_f32 and
mtts_plm_infer_mix_f32) - the oracle of mix_logprob_rows_kernel (csrc/sample.cu) and of MegaPLM.infer_mix.

Test infrastructure only: the mixture in fp64, the picks by the sampler's oracle (oracle/ref_sampling.py), the per-source
step logits by the reference restatement (oracle/ref_megatts2.py)."""
import numpy as np
import torch

from oracle import ref_megatts2 as R
from oracle import ref_sampling as RS


def mix_logprobs(rows, weights):
    """rows (K, V) logits of one utterance (fp32), weights (K,) -> l (V,) fp64: log sum_k w^_k softmax(rows[k]), with the
    contract's rules for NaN / -inf (no mass), +inf (all mass on the lowest +inf index), sources without a candidate (no
    contribution) and exactly one positive weight (the raw fp32 row)."""
    z = np.asarray(rows, dtype=np.float32)
    w = np.asarray(weights, dtype=np.float32).astype(np.float64)      # the device reads fp32 weights
    K, V = z.shape
    pos = np.nonzero(w > 0)[0]
    if pos.size == 1:
        return z[pos[0]].astype(np.float64)
    p = np.zeros(V)
    if pos.size:
        wn = w / w[pos].sum()
        for k in pos:
            zk = z[k].astype(np.float64)
            inf = np.nonzero(zk == np.inf)[0]
            if inf.size:
                p[inf[0]] += wn[k]
                continue
            cand = np.isfinite(zk)
            if not cand.any():
                continue
            e = np.exp(zk[cand] - zk[cand].max())
            p[cand] += wn[k] * e / e.sum()
    with np.errstate(divide="ignore"):
        return np.log(p)


def mix_pick(rows, weights, step=0, sampling=None, key=0):
    """The code the contract picks from rows (K, V) at AR step `step` -> (pick, relative gap of the two best fp64 scores;
    inf when the pick is not a score contest).  sampling None = greedy; else (temperature, top_k, top_p, seed)."""
    l = mix_logprobs(rows, weights)
    if sampling is None or float(np.float32(sampling[0])) == 0.0 or sampling[1] == 1:
        cand = np.nonzero(~np.isnan(l) & (l != -np.inf))[0]
        if not cand.size:
            return 0, np.inf
        if np.any(l == np.inf):
            return int(np.nonzero(l == np.inf)[0][0]), np.inf
        s = l[cand]
        best = int(cand[s == s.max()].min())
        if s.size < 2:
            return best, np.inf
        top2 = np.sort(s)[-2:]
        return best, (top2[1] - top2[0]) / max(1.0, abs(top2[1]))
    t, k, p, seed = sampling
    pick, s, _ = RS.sample_row(l.astype(np.float32), step, t, k, p, seed, key)
    if s is None or s.size < 2:
        return pick, np.inf
    top2 = np.sort(s)[-2:]
    return pick, (top2[1] - top2[0]) / max(1.0, abs(top2[1]))


def plm_infer_mix(sd, tc_latents, cfg, weights, sampling=None, keys=None, return_logits=False):
    """MegaPLM.infer_mix: K sources (B, T, tc_dim) share one code history; each step's per-source logits come from
    R.plm_step_logits and the code from mix_pick.  weights (B, K).  -> codes (B, T) [, logits (K, B, T, V), near-tie gaps
    (B, T)]."""
    K = len(tc_latents)
    B, T, _ = tc_latents[0].shape
    w = np.asarray(weights, dtype=np.float32).reshape(B, K)
    keys = np.arange(B) if keys is None else np.asarray(keys)
    codes = torch.full((B, 1), cfg["vq_bins"], dtype=torch.int64)
    all_logits, gaps = [], np.full((B, T), np.inf)
    for t in range(T):
        lg = torch.stack([R.plm_step_logits(sd, tc, codes, cfg) for tc in tc_latents])       # (K, B, V)
        all_logits.append(lg)
        picks = torch.zeros(B, dtype=torch.int64)
        for b in range(B):
            picks[b], gaps[b, t] = mix_pick(lg[:, b].numpy(), w[b], t, sampling, int(keys[b]))
        codes = torch.cat([codes, picks[:, None]], 1)
    out = codes[:, 1:]
    return (out, torch.stack(all_logits, 2), gaps) if return_logits else out
