"""torch CPU restatement of the duration mix (include/megatts2_b200.h, mtts_adm_readout_mix_f32 and
mtts_adm_infer_mix_f32) - the oracle of adm_readout_mix_kernel (csrc/ops.cu) and of MegaADM.infer_mix.

Test infrastructure only: each source's step is R.adm_infer's loop body (oracle/ref_megatts2.py: the ADM weights,
sine_pe_add, encoder) run in the dtype of the state dict and latents it is given, so fp64 inputs give the fp64 oracle and
fp32 inputs reproduce R.adm_infer's arithmetic step for step."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import ref_megatts2 as R


def sd64(sd):
    """A flat state dict in fp64, as an R.SD view."""
    return R.SD({k: v.double() for k, v in sd.items()})


def mix_readout(ys, weights):
    """ys (K,) readouts of one utterance, weights (K,) fp32 -> r, by the contract's rule: w^ = w / sum in fp32 (positive
    weights, k order), the first positive term w^ y, the later ones added in k order, the products and sums in the dtype
    of ys (the device uses fp32 fmaf).  Zero-weight sources are skipped whatever their y; without a positive weight
    r = 0.  With one positive weight w^ = 1 exactly, so r is that y, -0 included."""
    w = np.asarray(weights, dtype=np.float32)
    ys = torch.as_tensor(ys)
    pos = [k for k in range(len(w)) if w[k] > 0]
    if not pos:
        return torch.zeros((), dtype=ys.dtype)
    wsum = torch.zeros((), dtype=torch.float32)
    for k in pos:
        wsum = wsum + torch.tensor(w[k])                       # fp32, k order, as on the device
    r = None
    for k in pos:
        wn = (torch.tensor(w[k]) / wsum).to(ys.dtype)
        r = wn * ys[k] if r is None else r + wn * ys[k]
    return r


def adm_step(sd, tc_latent, p, t, cfg):
    """One body of R.adm_infer's loop: tc_latent (B, T, tc_dim), p (B, t+1, 1) the raw history -> y (B, 1, 1)."""
    w_dt, w_tc, w_out = sd("dt_linear_emb.weight"), sd("tc_linear_emb.weight"), sd("predict_layer.weight")
    dt_emb = F.linear(p, w_dt)
    tc_emb = F.linear(tc_latent[:, : t + 1], w_tc)
    x = R.sine_pe_add(torch.cat([tc_emb, dt_emb], -1), sd("pos_emb.alpha"))
    x = R.encoder(sd.sub("adm"), x, cfg["n_layers"], cfg["n_heads"], False)
    return F.linear(x, w_out)[:, -1:, :]


def adm_infer_mix(sd, tc_latents, cfg, weights, return_raw=False):
    """MegaADM.infer_mix: K sources (B, T, tc_dim) share one raw history; step t runs adm_step on each source with a
    positive weight in some row (every source when return_raw) and feeds back mix_readout per utterance.  weights (B, K)
    fp32.  -> durations (B, T, 1) int32 [, raw (B, T, 1), raw_src (K, B, T)]."""
    K = len(tc_latents)
    B, T, _ = tc_latents[0].shape
    dtype = tc_latents[0].dtype
    w = np.asarray(weights, dtype=np.float32).reshape(B, K)
    p = torch.zeros(B, 1, 1, dtype=dtype)
    raw_src = torch.full((K, B, T), float("nan"), dtype=dtype)
    for t in range(T):
        ys = {}
        for k in range(K):
            if return_raw or bool((w[:, k] > 0).any()):
                ys[k] = adm_step(sd, tc_latents[k], p, t, cfg)[:, 0, 0]
                raw_src[k, :, t] = ys[k]
        r = torch.zeros(B, dtype=dtype)
        for b in range(B):
            yb = torch.stack([ys[k][b] if k in ys else torch.zeros((), dtype=dtype) for k in range(K)])
            r[b] = mix_readout(yb, w[b])
        p = torch.cat([p, r.reshape(B, 1, 1)], 1)
    raw = p[:, 1:, :]
    dur = (raw + 0.5).to(torch.int32).clamp(1, 128)
    return (dur, raw, raw_src) if return_raw else dur
