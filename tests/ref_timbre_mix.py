"""torch CPU restatement of timbre interpolation (include/megatts2_b200.h, mtts_mix_layernorm_f32; MRTE.tc_latent_mix) -
the oracle of mix_layernorm_kernel (csrc/ops.cu) and of the timbre blend of Megatts.synthesize.

Test infrastructure only.  ``tc_latent_mix`` is R.mrte_tc_latent (oracle/ref_megatts2.py) split at the LayerNorm: the
phone encoder once (px), the mel encoder and the MHA per source (y_k), the w^-mix of the y_k, then LayerNorm and ReLU.
It runs in the dtype of the state dict it is given, so fp64 weights (ref_duration_mix.sd64) give the fp64 oracle."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import ref_megatts2 as R


def weight_rows(weights, K, B, T):
    """(K,), (B, K) or (B, T, K) weights -> (B, T, K) fp32 rows."""
    w = torch.as_tensor(np.asarray(weights, dtype=np.float32))
    if w.dim() == 1:
        w = w[None, None].expand(B, T, K)
    elif w.dim() == 2:
        w = w[:, None].expand(B, T, K)
    assert tuple(w.shape) == (B, T, K)
    return w


def normalised(w):
    """(..., K) fp32 weights -> w^ in fp64: the positive weights over their sum (zero, negative and NaN weights count as
    0).  A row without a positive weight is all zeros."""
    w = w.to(torch.float64)
    w = torch.where(w > 0, w, torch.zeros_like(w))
    s = w.sum(-1, keepdim=True)
    return torch.where(s > 0, w / torch.where(s > 0, s, torch.ones_like(s)), torch.zeros_like(w))


def mix_layernorm(ys, weights, gamma, beta, eps=1e-5, relu=True):
    """ys (K, B, T, C) and weights (K,), (B, K) or (B, T, K) -> post(LN(sum_k w^_k ys[k])) in fp64.  Sources without a
    positive weight are left out of the sum altogether (their values, NaN or inf included, never enter it)."""
    K, B, T, C = ys.shape
    wn = normalised(weight_rows(weights, K, B, T))
    m = torch.zeros(B, T, C, dtype=torch.float64)
    for k in range(K):
        on = wn[..., k] > 0
        if bool(on.any()):
            m = m + torch.where(on[..., None], wn[..., k:k + 1] * ys[k].to(torch.float64), torch.zeros_like(m))
    y = R.layer_norm(m, gamma.to(torch.float64), beta.to(torch.float64), eps)
    return F.relu(y) if relu else y


def attend(sd, phone, mels, cfg):
    """The pre-norm MRTE attention outputs (K, B, Tp, H) of the K mels, px computed once (R.mrte_tc_latent's steps)."""
    dt = sd("phone_embedding.word_embeddings.weight").dtype
    emb = F.embedding(phone, sd("phone_embedding.word_embeddings.weight"))
    x = R.sine_pe_add(emb, sd("phone_pos_embedding.alpha"))
    stride = cfg["mel_stride"]

    def middle(ls, y):
        return F.conv1d(y, sd("mel_encoder_middle_layer.weight"), sd("mel_encoder_middle_layer.bias"),
                        stride=stride, padding=stride // 2)
    px = R.encoder(sd.sub("phone_encoder"), x, cfg["content_layers"], cfg["content_heads"], True)
    ys = []
    for mel in mels:
        ctx = R.convnet_double(sd.sub("mel_encoder"), mel.to(dt).transpose(1, 2), cfg["mel_kernel"], cfg["mel_n_layer"],
                               cfg["mel_n_stack"], cfg["mel_n_block"], middle).transpose(1, 2)
        ys.append(R.mha(sd.sub("mha"), px, 1, kv_in=ctx))
    return torch.stack(ys)


def tc_latent_mix(sd, phone, mels, weights, cfg):
    """MRTE.tc_latent_mix: sd an R.SD view of the MRTE weights, phone (B, Tp), mels K tensors (B, Tm_k, 80), weights
    (K,), (B, K) or (B, Tp, K) -> (B, Tp, H) in the dtype of sd (the mix and the LayerNorm in fp64)."""
    ys = attend(sd, phone, mels, cfg)
    return mix_layernorm(ys, weights, sd("norm.weight"), sd("norm.bias")).to(ys.dtype)
