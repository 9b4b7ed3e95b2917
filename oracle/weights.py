"""Deterministic, reference-free weights for the oracle / parity tests / bench.

TEST INFRASTRUCTURE (see oracle/__init__.py).  No checkpoint of the reference
exists anywhere (infer.py:5-10 points at the author's local files), so parity is
checked on seeded random weights.  Every tensor is a pure function of
(base_seed, state_dict key, shape): the same values are produced wherever they
are built (oracle/make_golden.py loads them into the real reference via
load_state_dict; the tests only need this module).

Key sets follow the reference's state_dict layout (SURVEY.md §8b); a golden test
pins them against the real reference's ``state_dict().keys()``.
"""
import math
import zlib

import torch

# --- architecture constants: configs/config_{gan,plm,adm}.yaml of the reference
G_CFG = dict(
    mel_bins=80, hidden=512, mel_kernel=3, mel_stride=16, mel_n_layer=5, mel_n_stack=5,
    mel_n_block=2, content_ff=1024, content_heads=2, content_layers=8, phone_vocab=320,
    vq_mel_bins=20, vq_stride=8, vq_hidden=384, vq_kernel=5, vq_n_layer=3, vq_n_stack=5,
    vq_n_block=2, vq_bins=1024, vq_dim=256, dec_kernel=5, dec_hidden=512, dec_n_stack=4,
    dec_n_block=2)
PLM_CFG = dict(n_layers=12, n_heads=16, vq_dim=512, tc_latent_dim=512, vq_bins=1024)
ADM_CFG = dict(n_layers=8, n_heads=8, emb_dim=256, tc_latent_dim=512, tc_emb_dim=512)
HIFIGAN_CFG = dict(
    in_channels=80, upsample_initial_channel=512, upsample_factors=(8, 8, 2, 2),
    upsample_kernel_sizes=(16, 16, 4, 4), resblock_kernel_sizes=(3, 7, 11),
    resblock_dilation_sizes=((1, 3, 5), (1, 3, 5), (1, 3, 5)), inference_padding=5)


def _conv(spec, p, cout, cin, k, bias=True):
    spec[p + ".weight"] = (cout, cin, k)
    if bias:
        spec[p + ".bias"] = (cout,)


def _lin(spec, p, cout, cin, bias=True):
    spec[p + ".weight"] = (cout, cin)
    if bias:
        spec[p + ".bias"] = (cout,)


def _ln(spec, p, c):
    spec[p + ".weight"] = (c,)
    spec[p + ".bias"] = (c,)


def _res_stack(spec, p, c, k, n_stacks, n_blocks):
    for s in range(n_stacks):
        for b in range(n_blocks):
            q = f"{p}.conv_stacks.{s}.blocks.{b}"
            _conv(spec, q + ".conv", c, c, k)
            _ln(spec, q + ".norm", c)


def _encoder(spec, p, n_layers, d, ff, conv_ff):
    for i in range(n_layers):
        q = f"{p}.layers.{i}"
        _ln(spec, q + ".norm1", d)
        _ln(spec, q + ".norm2", d)
        for w in ("w_q", "w_k", "w_v"):
            _lin(spec, f"{q}.attn.{w}", d, d)
        _lin(spec, q + ".attn.out_proj.0", d, d)
        if conv_ff:
            _conv(spec, q + ".ff.0", ff, d, 5)
            _conv(spec, q + ".ff.2", d, ff, 5)
        else:
            _lin(spec, q + ".ff.0", ff, d)
            _lin(spec, q + ".ff.3", d, ff)


def g_spec(cfg=G_CFG):
    """Key -> shape of MegaG.state_dict() (models/megatts2.py:30-54 with
    configs/config_gan.yaml:38-76), in the reference's registration order."""
    c = cfg
    H = c["hidden"]
    s = {}
    s["mrte.phone_embedding.word_embeddings.weight"] = (c["phone_vocab"], H)
    s["mrte.phone_pos_embedding.alpha"] = (1,)
    _conv(s, "mrte.mel_encoder_middle_layer", H, H, c["mel_stride"] + 1)
    _conv(s, "mrte.mel_encoder.first_layer", H, c["mel_bins"], c["mel_kernel"])
    for l in range(c["mel_n_layer"]):
        p = f"mrte.mel_encoder.layers.{l}"
        _res_stack(s, p + ".conv_stack1", H, c["mel_kernel"], c["mel_n_stack"], c["mel_n_block"])
        _conv(s, p + ".middle_layer", H, H, c["mel_stride"] + 1)   # alias of mel_encoder_middle_layer
        _res_stack(s, p + ".conv_stack2", H, c["mel_kernel"], c["mel_n_stack"], c["mel_n_block"])
    _conv(s, "mrte.mel_encoder.last_layer", H, H, c["mel_kernel"])
    _encoder(s, "mrte.phone_encoder", c["content_layers"], H, c["content_ff"], True)
    for w in ("w_q", "w_k", "w_v"):
        _lin(s, f"mrte.mha.{w}", H, H)
    _lin(s, "mrte.mha.out_proj.0", H, H)
    _ln(s, "mrte.norm", H)
    V = c["vq_hidden"]
    _conv(s, "vqpe.convnet.first_layer", V, c["vq_mel_bins"], c["vq_kernel"])
    for l in range(c["vq_n_layer"]):
        p = f"vqpe.convnet.layers.{l}"
        _res_stack(s, p + ".conv_stack1", V, c["vq_kernel"], c["vq_n_stack"], c["vq_n_block"])
        _res_stack(s, p + ".conv_stack2", V, c["vq_kernel"], c["vq_n_stack"], c["vq_n_block"])
    _conv(s, "vqpe.convnet.last_layer", c["vq_dim"], V, c["vq_kernel"])
    cb = "vqpe.vq.vq.layers.0._codebook"
    s[cb + ".inited"] = (1,)
    s[cb + ".cluster_size"] = (c["vq_bins"],)
    s[cb + ".embed"] = (c["vq_bins"], c["vq_dim"])
    s[cb + ".embed_avg"] = (c["vq_bins"], c["vq_dim"])
    D = c["dec_hidden"]
    _conv(s, "decoder.first_layer", D, H + c["vq_dim"], c["dec_kernel"])
    _res_stack(s, "decoder.conv_stack", D, c["dec_kernel"], c["dec_n_stack"], c["dec_n_block"])
    _conv(s, "decoder.last_layer", c["mel_bins"], D, c["dec_kernel"])
    return s


def plm_spec(cfg=PLM_CFG):
    """MegaPLM.state_dict() (models/megatts2.py:120-146)."""
    d = cfg["vq_dim"] + cfg["tc_latent_dim"]
    s = {}
    _encoder(s, "plm", cfg["n_layers"], d, 4 * d, False)
    _lin(s, "predict_layer", cfg["vq_bins"], d, bias=False)
    s["pos.alpha"] = (1,)
    s["pc_embedding.weight"] = (cfg["vq_bins"] + 2, cfg["vq_dim"])
    return s


def adm_spec(cfg=ADM_CFG):
    """MegaADM.state_dict() (models/megatts2.py:201-231)."""
    d = cfg["emb_dim"] + cfg["tc_emb_dim"]
    s = {}
    _encoder(s, "adm", cfg["n_layers"], d, 4 * cfg["emb_dim"], False)
    _lin(s, "dt_linear_emb", cfg["emb_dim"], 1, bias=False)
    _lin(s, "tc_linear_emb", cfg["tc_emb_dim"], cfg["tc_latent_dim"], bias=False)
    s["pos_emb.alpha"] = (1,)
    _lin(s, "predict_layer", 1, d, bias=False)
    return s


def hifigan_spec(cfg=HIFIGAN_CFG):
    """HiFi-GAN V1 generator after weight-norm folding (speechbrain
    HifiganGenerator [memory]; SURVEY.md §8c).  ConvTranspose1d weights are
    (Cin, Cout, k) as in torch."""
    s = {}
    ch = cfg["upsample_initial_channel"]
    _conv(s, "conv_pre", ch, cfg["in_channels"], 7)
    nk = len(cfg["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(cfg["upsample_factors"], cfg["upsample_kernel_sizes"])):
        cin, cout = ch // (2 ** i), ch // (2 ** (i + 1))
        s[f"ups.{i}.weight"] = (cin, cout, k)
        s[f"ups.{i}.bias"] = (cout,)
        for j, rk in enumerate(cfg["resblock_kernel_sizes"]):
            for m in range(len(cfg["resblock_dilation_sizes"][j])):
                _conv(s, f"resblocks.{i * nk + j}.convs1.{m}", cout, cout, rk)
                _conv(s, f"resblocks.{i * nk + j}.convs2.{m}", cout, cout, rk)
    _conv(s, "conv_post", 1, ch // (2 ** len(cfg["upsample_factors"])), 7)
    return s


def _gen(seed, key):
    g = torch.Generator()
    g.manual_seed((seed * 1000003 + zlib.crc32(key.encode())) & 0x7FFFFFFFFFFF)
    return g


def make_state_dict(spec, seed, transposed_fan_in=()):
    """Fill a key->shape spec with seeded fp32 values.

    * ``*norm*.weight`` ~ 1 + 0.1 N(0,1); ``*norm*.bias`` ~ 0.1 N(0,1)
    * ``alpha`` = 1 (embedding.py:58)
    * embeddings / codebook ``embed`` ~ N(0,1); ``inited`` = 1 (else the reference
      runs k-means on first call even in eval, core_vq.py:141-149)
    * other >=2-D weights ~ U(-1/sqrt(fan_in), +1/sqrt(fan_in)); 1-D biases ~ 0.05 N(0,1)
    """
    sd = {}
    for key, shape in spec.items():
        g = _gen(seed, key)
        leaf = key.rsplit(".", 1)[-1]
        if key.endswith("middle_layer.weight") or key.endswith("middle_layer.bias"):
            # the 5 ConvNetDoubleLayer.middle_layer entries alias ONE conv (mrte.py:101-118)
            if key.startswith("mrte.mel_encoder.layers."):
                sd[key] = sd["mrte.mel_encoder_middle_layer." + leaf]
                continue
        if leaf == "alpha":
            t = torch.ones(shape)
        elif leaf == "inited":
            t = torch.ones(shape)
        elif leaf == "cluster_size":
            t = torch.ones(shape)
        elif leaf == "embed_avg":
            t = sd[key[:-len("_avg")]].clone()
        elif leaf == "embed" or "embedding" in key:
            t = torch.randn(shape, generator=g)
        elif "norm" in key and leaf == "weight":
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif "norm" in key and leaf == "bias":
            t = 0.1 * torch.randn(shape, generator=g)
        elif len(shape) >= 2:
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            if key.startswith("ups."):           # ConvTranspose1d (Cin, Cout, k)
                fan_in = shape[0] * shape[2]
            b = 1.0 / math.sqrt(fan_in)
            t = (torch.rand(shape, generator=g) * 2.0 - 1.0) * b
        else:
            t = 0.05 * torch.randn(shape, generator=g)
        sd[key] = t.to(torch.float32).contiguous()
    return sd


def g_state_dict(seed=0):
    return make_state_dict(g_spec(), seed)


def plm_state_dict(seed=1, logit_gain=4.0):
    """``logit_gain`` scales predict_layer so that greedy ids are diverse on random
    weights (default init gives ~3 distinct ids in 48 steps, SURVEY.md §7.2)."""
    sd = make_state_dict(plm_spec(), seed)
    sd["predict_layer.weight"] = sd["predict_layer.weight"] * logit_gain
    return sd


def adm_state_dict(seed=2, dur_gain=12.0, dt_scale=0.02, dur_offset=6.0):
    """Random-weight ADM shaped so the AR regression is stable and non-degenerate:
    ``dt_scale`` shrinks dt_linear_emb (fan_in 1; raw float predictions are fed back,
    models/megatts2.py:265,273), ``dur_gain`` scales predict_layer, and ``dur_offset`` is
    injected through the last layer's ff.3.bias along predict_layer's direction so the
    predicted durations spread over ~[1,12] instead of sitting at the clamp floor."""
    sd = make_state_dict(adm_spec(), seed)
    sd["dt_linear_emb.weight"] = sd["dt_linear_emb.weight"] * dt_scale
    w = sd["predict_layer.weight"] * dur_gain
    sd["predict_layer.weight"] = w
    last = ADM_CFG["n_layers"] - 1
    sd[f"adm.layers.{last}.ff.3.bias"] = sd[f"adm.layers.{last}.ff.3.bias"] + dur_offset * w[0] / (w[0] @ w[0])
    return sd


def hifigan_state_dict(seed=3):
    return make_state_dict(hifigan_spec(), seed)
