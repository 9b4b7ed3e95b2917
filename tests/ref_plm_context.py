"""fp32 / fp64 restatement of the prosody LM's in-context decode (include/megatts2_b200.h, in-context prompting) - the
oracle of MegaPLM.infer / infer_causal with a context.

Test infrastructure only.  Both forms are written from oracle/ref_megatts2.py: the non-causal step is R.plm_step_logits over
the concatenated latents and codes, the causal step is the last row of R.plm_forward over the concatenation.  Target step
j of a P-row context is the reference loop's step P + j; a sampled draw is keyed by j (oracle/ref_sampling.py)."""
import torch

from oracle import ref_megatts2 as R
from oracle import ref_sampling as RS


def sd_as(sd, dtype):
    """A flat state_dict with every floating tensor in ``dtype`` (fp64 for the fp64 restatement)."""
    return {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}


def concat(ctx_tc, ctx_codes, tc, vq_bins):
    """(latents (B, P+T, tc_dim), code history [BOS, ctx_codes] (B, P+1)); a Bc = 1 context is broadcast over B."""
    B = tc.shape[0]
    ctx_tc = ctx_tc.to(tc.dtype).expand(B, -1, -1)
    ctx_codes = ctx_codes.to(torch.int64).expand(B, -1)
    bos = torch.full((B, 1), vq_bins, dtype=torch.int64)
    return torch.cat([ctx_tc, tc], 1), torch.cat([bos, ctx_codes], 1)


def step_logits(sd, lat, codes, cfg, causal):
    """Logits (B, V) of the step whose code history is ``codes`` (B, s) over latents lat[:, :s]."""
    if not causal:
        return R.plm_step_logits(R.SD(sd), lat, codes, cfg)
    s = codes.shape[1]
    pcodes = torch.cat([codes, codes[:, :1]], 1)                          # forward() drops the last column
    lens = torch.full((codes.shape[0],), s, dtype=torch.int32)
    return R.plm_forward(R.SD(sd), lat[:, :s], pcodes, lens, cfg)[0][:, -1]


def plm_infer_ctx(sd, ctx_tc, ctx_codes, tc, cfg, causal=False, sampling=None, keys=None, return_logits=False):
    """The decode of the target tc (B, T, tc_dim) after the context (ctx_tc (Bc, P, tc_dim), ctx_codes (Bc, P)), in the dtype
    of ``sd`` and ``tc``: greedy, or with ``sampling`` = (temperature, top_k, top_p, seed) and row ``keys``.  causal=False is
    MegaPLM.infer over the concatenation with the first P codes teacher-forced, causal=True its training-mode form.  P = 0
    is R.plm_infer / R.plm_infer_causal.  -> codes (B, T) [, logits (B, T, V)]."""
    B, T, _ = tc.shape
    lat, codes = concat(ctx_tc, ctx_codes, tc, cfg["vq_bins"])
    keys = list(range(B)) if keys is None else [int(k) for k in keys]
    all_logits = []
    for j in range(T):
        lg = step_logits(sd, lat, codes, cfg, causal)
        all_logits.append(lg)
        if sampling is None:
            pick = lg.argmax(-1)
        else:
            t, k, p, seed = sampling
            pick = torch.tensor([RS.sample_row(lg[b].float().numpy(), j, t, k, p, seed, keys[b])[0] for b in range(B)])
        codes = torch.cat([codes, pick.reshape(B, 1)], 1)
    out = codes[:, codes.shape[1] - T:]
    return (out, torch.stack(all_logits, 1)) if return_logits else out


def causal_logits_on(sd, ctx_tc, ctx_codes, tc, codes, cfg):
    """The teacher-forced causal forward (R.plm_forward) over [context; target] evaluated on the target codes ``codes``
    (B, T): the logits of the target rows, (B, T, V), in one pass."""
    T = tc.shape[1]
    lat, hist = concat(ctx_tc, ctx_codes, tc, cfg["vq_bins"])
    pcodes = torch.cat([hist, codes.to(torch.int64)], 1)                 # forward() drops the last column
    lens = torch.full((tc.shape[0],), lat.shape[1], dtype=torch.int32)
    return R.plm_forward(R.SD(sd), lat, pcodes, lens, cfg)[0][:, -T:]
