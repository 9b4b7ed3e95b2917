"""GPU: the wgmma engine (both operand formats: bf16x3 = engine 1, f16x2 = engine 2) against fp64 and against the
exact FFMA engine / golden ids."""
import math

import pytest
import torch

import helpers
from megatts2_b200 import pack

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
DEV = "cuda"
ENGINES = [pytest.param(1, id="bf16x3"), pytest.param(2, id="f16x2")]


def fmt_of(engine):
    return pack.engine_fmt(engine)


def gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


CASES = [
    dict(M=128, K=64, N=128),
    dict(M=256, K=1024, N=1024, bias=True),
    dict(M=4096, K=1024, N=3072, bias=True),
    dict(M=1000, K=1024, N=4096, bias=True, relu=True),            # M tail
    dict(M=2048, K=4096, N=1024, bias=True, res=True),
    dict(M=300, K=768, N=2304, bias=True, plan=dict(BN=64)),       # ADM qkv
    dict(M=640, K=72, N=192, plan=dict(BN=32)),                    # K tail, N not a multiple of 128
    dict(M=129, K=1024, N=1024, res=True),
    dict(M=8192, K=4096, N=1024, bias=True, res=True, plan=dict(BN=128)),   # long K
    dict(M=5000, K=1024, N=768, bias=True, relu=True, plan=dict(BN=128)),   # M tail
    dict(M=16384, K=80, N=512, bias=True, plan=dict(BN=128)),      # K tail inside the second 64-wide slab
]


def _ids(c):
    return "-".join(f"{k}{v}" for k, v in c.items() if k != "plan")


def assert_plan(c, B, T, Cin, Cout, k, dil, engine):
    """the plan a case exists to reach (key `plan`), as the dispatcher reports it for the 132 SMs of an H100 SXM
    (mtts_tc_plan_query; no partial-sum space: these calls cannot split K)"""
    import ctypes
    from megatts2_b200 import _lib as L
    if "plan" not in c:
        return
    out = (ctypes.c_int32 * 5)()
    L.check(L.lib().mtts_tc_plan_query(132, B, T, Cin, Cout, k, dil, fmt_of(engine), 0, 0, out))
    got = dict(BN=out[0], splits=out[1], halo=out[3], swb=out[4])
    assert {key: got[key] for key in c["plan"]} == c["plan"], (c, got)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("c", CASES, ids=_ids)
def test_linear_tc_vs_fp64(c, engine):
    from megatts2_b200 import ops
    assert_plan(c, 1, c["M"], c["K"], c["N"], 1, 1, engine)
    g = gen(c["M"] + c["K"] + c["N"])
    x = torch.randn(c["M"], c["K"], generator=g) * 2
    w = torch.randn(c["N"], c["K"], generator=g) / math.sqrt(c["K"])
    b = torch.randn(c["N"], generator=g) if c.get("bias") else None
    r = torch.randn(c["M"], c["N"], generator=g) if c.get("res") else None
    ref = x.double() @ w.double().t()
    if b is not None:
        ref = ref + b.double()
    if c.get("relu"):
        ref = torch.relu(ref)
    if r is not None:
        ref = ref + r.double()
    y = ops.linear_tc(x.to(DEV), pack.pack_tc_planes(w.to(DEV), fmt_of(engine)), b.to(DEV) if b is not None else None,
                      res=r.to(DEV) if r is not None else None, post_act=1 if c.get("relu") else 0)
    torch.cuda.synchronize()
    err = (y.cpu().double() - ref).abs().max().item()
    # fp32-grade: the split drops O(2^-24) terms; accumulation is fp32 in the wgmma register accumulators
    assert err < 3e-5 * max(1.0, ref.abs().max().item()), err
    # and it must be much closer to fp64 than a single-pass bf16 product could be (~4e-3 relative)
    y_ffma = ops.linear(x.to(DEV), pack.pack_linear(w).to(DEV), b.to(DEV) if b is not None else None,
                        res=r.to(DEV) if r is not None else None, post_act=1 if c.get("relu") else 0)
    err_ffma = (y_ffma.cpu().double() - ref).abs().max().item()
    print(f"tc err {err:.3e}  ffma err {err_ffma:.3e}")
    assert err < 20 * max(err_ffma, 1e-7)


def test_split_planes_are_exact():
    w = torch.randn(257, 96, generator=gen(1)) * 3
    p = pack.pack_tc_planes(w).float()
    assert (p.sum(0) - w).abs().max().item() <= 2.0 ** -22 * w.abs().max().item()


@pytest.mark.parametrize("engine", ENGINES)
def test_device_packing_equals_host_packing(engine):
    """Weights are re-laid out and split by the library's own kernels on the device (mtts_copy_strided_f32 +
    mtts_split_planes_f32); the torch implementation in pack.py (CPU tensors) is the layout specification: bit-equal."""
    fmt = fmt_of(engine)
    g = gen(17)
    w2, wc, wt = torch.randn(300, 136, generator=g), torch.randn(96, 64, 7, generator=g), torch.randn(64, 32, 16, generator=g)
    bt = torch.randn(32, generator=g)
    for host, dev in ((pack.pack_linear(w2), pack.pack_linear(w2.to(DEV))),
                      (pack.pack_conv(wc), pack.pack_conv(wc.to(DEV))),
                      (pack.pack_qkv(w2[:100], w2[100:200], w2[200:]), pack.pack_qkv(w2[:100].to(DEV), w2[100:200].to(DEV), w2[200:].to(DEV))),
                      (pack.pack_tc_planes(w2, fmt), pack.pack_tc_planes(w2.to(DEV), fmt)),
                      (pack.pack_conv_tc_planes(wc, fmt), pack.pack_conv_tc_planes(wc.to(DEV), fmt)),
                      (pack.cat_vectors(bt, bt * 2), pack.cat_vectors(bt.to(DEV), bt.to(DEV) * 2)),
                      (pack.cat_rows(w2[:7], w2[7:20]), pack.cat_rows(w2[:7].to(DEV), w2[7:20].to(DEV)))):
        assert host.shape == dev.shape and host.dtype == dev.dtype
        assert torch.equal(host.view(torch.int16) if host.dtype != torch.float32 else host,
                           dev.cpu().view(torch.int16) if dev.dtype != torch.float32 else dev.cpu())
    (wh, bh), (wd, bd) = pack.pack_conv_transpose(wt, bt, 8), pack.pack_conv_transpose(wt.to(DEV), bt.to(DEV), 8)
    assert torch.equal(wh, wd.cpu()) and torch.equal(bh, bd.cpu())
    assert torch.equal(pack.pack_conv_transpose_tc_planes(wh, fmt).view(torch.int16),
                       pack.pack_conv_transpose_tc_planes(wd, fmt).cpu().view(torch.int16))


def test_f16x2_range_guard():
    """An activation beyond the fp16 range cannot be split: the result is poisoned (non-finite) and the flag registered
    with mtts_tc_overflow_bind is raised; in range, the flag stays clear."""
    from megatts2_b200 import ops
    dev = torch.device(DEV)
    ops.tc_overflow(dev)                                            # clear
    x = torch.randn(256, 128, generator=gen(2)).to(DEV)
    w = pack.pack_tc_planes((torch.randn(128, 128, generator=gen(3)) / 11).to(DEV), pack.FMT_F16X2)
    y = ops.linear_tc(x * 6e4 / x.abs().max(), w)
    assert torch.isfinite(y).all() and not ops.tc_overflow(dev)
    x[5, 7] = 7.0e4
    y = ops.linear_tc(x, w)
    assert not torch.isfinite(y[5]).all()
    assert torch.isfinite(y[6]).all()
    assert ops.tc_overflow(dev) and not ops.tc_overflow(dev)        # raised once, reset by the read
    # the bf16x3 format has the fp32 range
    y3 = ops.linear_tc(x, pack.pack_tc_planes((torch.randn(128, 128, generator=gen(3)) / 11).to(DEV), pack.FMT_BF16X3))
    assert torch.isfinite(y3).all() and not ops.tc_overflow(dev)


@pytest.mark.parametrize("engine", ENGINES)
def test_plm_tc_engine_matches_golden_ids(golden, weights_cpu, engine):
    g = golden("plm")
    plm = helpers.build_plm(weights_cpu("plm"), DEV)
    plm.plm.engine = engine
    big = torch.cat([g["tc8"]] * 8, 0).to(DEV)                    # B = 16 so that M = B*(t+1) crosses 128
    ids, logits = plm.infer(big, return_logits=True)
    assert torch.equal(ids.cpu(), torch.cat([g["ids"]] * 8, 0)), "PLM ids must stay bit-exact on the tensor-core engine"
    assert (logits.cpu() - torch.cat([g["logits"]] * 8, 0)).abs().max().item() < 2e-3
    plm.plm.engine = 0
    ids0 = plm.infer(big)
    assert torch.equal(ids0, ids)


@pytest.mark.parametrize("engine", ENGINES)
def test_encoder_tc_vs_ffma(weights_cpu, engine):
    from megatts2_b200.modules.transformer import run_encoder
    plm = helpers.build_plm(weights_cpu("plm"), DEV)
    # (8, 40): every dense layer is under-filled -> split-K at full tile width; (16, 64): only the N = 1024 layers;
    # (64, 40): full grids (CTA pairs); (5, 33): ragged rows
    for i, (B, T) in enumerate([(8, 40), (16, 64), (64, 40), (5, 33)]):
        x = torch.randn(B, T, 1024, generator=gen(3 + i)).to(DEV)
        plm.plm.engine = 0
        y0 = plm.plm(x)
        plm.plm.engine = engine
        y1 = plm.plm(x)
        assert (y0 - y1).abs().max().item() < 5e-4, (B, T)
        assert torch.equal(y1, plm.plm(x)), "the split-K reduction order is fixed: bit-reproducible"
        l1 = run_encoder(plm.plm, list(plm.plm.layers), x, last_row_only=True)
        assert (l1[:, 0] - y0[:, -1]).abs().max().item() < 5e-4, (B, T)


# ------------------------------------------------------------------ tensor-core convolution engine
CONV_TC_CASES = [
    dict(B=2, T=500, Cin=512, Cout=512, k=3, pre=1),                                   # MRTE ConvBlock
    dict(B=2, T=300, Cin=384, Cout=384, k=5, pre=1),                                   # VQPE ConvBlock (Cin % 64 == 0)
    dict(B=2, T=1000, Cin=256, Cout=256, k=11, dil=5, pad_mode=1, pre=2, res=True),    # HiFi-GAN stage 1
    dict(B=3, T=777, Cin=128, Cout=128, k=3, dil=3, pad_mode=1, pre=2),                # stage 2, ragged tile
    # C = 64 at 32 tiles: plain BN = 32 (the fill rule narrows the tile)
    dict(B=2, T=2000, Cin=64, Cout=64, k=7, dil=3, pad_mode=1, pre=2, res=True, acc=True, scale=1 / 3, plan=dict(BN=32, halo=0)),
    dict(B=2, T=3000, Cin=32, Cout=32, k=3, pad_mode=1, pre=2, plan=dict(BN=32, swb=64, halo=1)),
    dict(B=2, T=1500, Cin=32, Cout=32, k=11, dil=1, pad_mode=1, pre=2, res=True),
    dict(B=2, T=64, Cin=512, Cout=1024, k=5, post=1),                                  # conv-FF first conv
    dict(B=2, T=64, Cin=1024, Cout=512, k=5, res=True),                                # conv-FF second conv
    dict(B=1, T=130, Cin=96, Cout=160, k=3, pad_mode=2),                               # odd sizes: K and N tails
    # full-machine grids (>= 132 tiles), long sequences: the halo form
    dict(B=4, T=5000, Cin=64, Cout=64, k=7, dil=3, pad_mode=1, pre=2, res=True, plan=dict(BN=64, halo=1)),
    dict(B=4, T=5000, Cin=64, Cout=64, k=11, dil=5, pad_mode=1, pre=2, res=True, acc=True, scale=1 / 3, plan=dict(BN=64, halo=1)),
    dict(B=4, T=5000, Cin=64, Cout=64, k=3, dil=1, pad_mode=1, pre=2, plan=dict(BN=64, halo=1)),
    dict(B=4, T=5001, Cin=32, Cout=32, k=11, dil=5, pad_mode=1, pre=2, res=True, plan=dict(BN=32, swb=64, halo=1)),
    dict(B=4, T=5000, Cin=32, Cout=32, k=3, dil=1, pad_mode=1, pre=2, plan=dict(BN=32, swb=64, halo=1)),
    dict(B=4, T=4999, Cin=32, Cout=32, k=7, dil=3, pad_mode=0, plan=dict(BN=32, swb=64, halo=1)),
    # BN = 128 tiles (Cout >= 256 and enough tiles to fill the machine)
    dict(B=8, T=2000, Cin=256, Cout=256, k=7, dil=3, pad_mode=1, pre=2, res=True, acc=True, scale=1 / 3, plan=dict(BN=128)),
    dict(B=8, T=1001, Cin=512, Cout=512, k=3, pre=1, post=1, plan=dict(BN=128)),
    dict(B=16, T=700, Cin=192, Cout=768, k=5, pad_mode=2, plan=dict(BN=128)),
]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", CONV_TC_CASES, ids=_ids)
def test_conv_tc_vs_fp64(case, engine):
    import torch.nn.functional as F
    from megatts2_b200 import ops
    c = dict(dil=1, pad_mode=0, pre=0, post=0, res=False, acc=False, scale=1.0)
    c.update(case)
    k, dil = c["k"], c["dil"]
    pad = dil * (k - 1) // 2
    assert_plan(c, c["B"], c["T"], c["Cin"], c["Cout"], k, dil, engine)
    g = gen(sum(v if isinstance(v, int) else 1 for key, v in case.items() if key != "plan"))
    x = torch.randn(c["B"], c["T"], c["Cin"], generator=g)
    w = torch.randn(c["Cout"], c["Cin"], k, generator=g) / math.sqrt(c["Cin"] * k)
    b = torch.randn(c["Cout"], generator=g)
    xin = F.leaky_relu(x, 0.1) if c["pre"] == 2 else (F.relu(x) if c["pre"] == 1 else x)
    xt = xin.transpose(1, 2).double()
    if c["pad_mode"] != 0:
        xt = F.pad(xt, (pad, pad), mode={1: "reflect", 2: "replicate"}[c["pad_mode"]])
        ref = F.conv1d(xt, w.double(), b.double(), dilation=dil)
    else:
        ref = F.conv1d(xt, w.double(), b.double(), dilation=dil, padding=pad)
    ref = ref.transpose(1, 2)
    if c["post"] == 1:
        ref = torch.relu(ref)
    res = torch.randn(ref.shape, generator=g) if c["res"] else None
    y0 = torch.randn(ref.shape, generator=g) if c["acc"] else None
    if res is not None:
        ref = ref + res.double()
    ref = ref * c["scale"]
    if y0 is not None:
        ref = ref + y0.double()
    kw = dict(k=k, dil=dil, pad=pad, pad_mode=c["pad_mode"], pre_act=c["pre"], pre_slope=0.1, post_act=c["post"],
              res=res.to(DEV) if res is not None else None, out_scale=c["scale"], accumulate=c["acc"])
    y_tc = ops.conv1d(x.to(DEV), pack.pack_conv(w).to(DEV), b.to(DEV), out=y0.clone().to(DEV) if y0 is not None else None,
                      w_tc=pack.pack_conv_tc_planes(w.to(DEV), fmt_of(engine)), **kw)
    y_ff = ops.conv1d(x.to(DEV), pack.pack_conv(w).to(DEV), b.to(DEV), out=y0.clone().to(DEV) if y0 is not None else None, **kw)
    torch.cuda.synchronize()
    e_tc = (y_tc.cpu().double() - ref).abs().max().item()
    e_ff = (y_ff.cpu().double() - ref).abs().max().item()
    print(f"conv tc err {e_tc:.3e}  ffma err {e_ff:.3e}")
    assert e_tc < 3e-5 * max(1.0, ref.abs().max().item())
    assert e_tc < 10 * max(e_ff, 1e-7)


def test_conv_tc_leaky_post_activation_matches_ffma():
    """post_act = LEAKY carries its slope on BOTH engines (ADVICE r1: the tensor-core epilogue used slope 0)."""
    from megatts2_b200 import _lib as L
    from megatts2_b200 import ops
    g = gen(91)
    x = torch.randn(2, 400, 64, generator=g).to(DEV)
    w = torch.randn(64, 64, 3, generator=g) / 14
    kw = dict(k=3, pad=1, post_act=L.ACT_LEAKY, post_slope=0.2)
    y0 = ops.conv1d(x, pack.pack_conv(w.to(DEV)), **kw)
    assert (y0 < 0).any()
    for engine in (1, 2):
        y1 = ops.conv1d(x, pack.pack_conv(w.to(DEV)), w_tc=pack.pack_conv_tc_planes(w.to(DEV), fmt_of(engine)), **kw)
        assert (y1 - y0).abs().max().item() < 1e-5


@pytest.mark.parametrize("engine", ENGINES)
def test_conv_stacks_tc_vs_oracle(weights_cpu, engine):
    """Tensor-core conv engine inside the drivers (shapes large enough to be eligible) vs the CPU oracle."""
    from oracle import ref_megatts2 as R
    from oracle import weights as W
    G = helpers.build_g(weights_cpu("g"), DEV)
    mel = torch.randn(4, 203, 80, generator=gen(61)) * 2 - 4
    sd = R.SD(weights_cpu("g"), "vqpe.")
    _, _, _, codes_ref, ze_ref = R.vqpe_forward(sd, mel, W.G_CFG)
    for m in (G.mrte.mel_encoder, G.mrte.phone_encoder, G.decoder):
        m.engine = engine
    for eng in (engine, 0):
        G.vqpe.convnet.engine = eng
        zq, _, _, codes = G.vqpe(mel.to(DEV))
        assert torch.equal(codes.cpu(), codes_ref), f"VQ codes differ on engine {eng}"
    phone = torch.randint(0, 320, (2, 16), generator=gen(62))
    melp = torch.randn(2, 300, 80, generator=gen(63)) * 2 - 4
    tc_ref, ctx_ref, _ = R.mrte_tc_latent(R.SD(weights_cpu("g"), "mrte."), phone, melp, W.G_CFG)
    tc = G.mrte.tc_latent(phone.to(DEV), melp.to(DEV))
    assert (tc.cpu() - tc_ref).abs().max().item() < 2e-4
    x = torch.randn(2, 768, 140, generator=gen(64))
    dec_ref = R.convnet(R.SD(weights_cpu("g"), "decoder."), x, 5, 4, 2)
    assert (G.decoder(x.to(DEV)).cpu() - dec_ref).abs().max().item() < 5e-4


@pytest.mark.parametrize("engine", ENGINES)
def test_hifigan_full_grid_vs_oracle(weights_cpu, engine):
    """B*L large enough that every stage launches full-machine grids inside the fused ResBlock flow."""
    from oracle import ref_megatts2 as R
    from oracle import weights as W
    hifi = helpers.build_hifigan(weights_cpu("hifigan"), DEV)
    mel = torch.randn(4, 80, 64, generator=gen(66)) * 2 - 4
    ref = R.hifigan_generator(weights_cpu("hifigan"), mel, W.HIFIGAN_CFG)
    hifi.generator.engine = engine
    w1 = hifi.decode_batch(mel.to(DEV))
    assert (w1.cpu() - ref).abs().max().item() < 1e-4


@pytest.mark.parametrize("engine", ENGINES)
def test_hifigan_tc_vs_oracle(weights_cpu, engine):
    from oracle import ref_megatts2 as R
    from oracle import weights as W
    hifi = helpers.build_hifigan(weights_cpu("hifigan"), DEV)
    mel = torch.randn(2, 80, 30, generator=gen(65)) * 2 - 4
    ref = R.hifigan_generator(weights_cpu("hifigan"), mel, W.HIFIGAN_CFG)
    hifi.generator.engine = engine
    w1 = hifi.decode_batch(mel.to(DEV))
    hifi.generator.engine = 0
    w0 = hifi.decode_batch(mel.to(DEV))
    assert (w1.cpu() - ref).abs().max().item() < 1e-4
    assert (w0.cpu() - ref).abs().max().item() < 1e-4
