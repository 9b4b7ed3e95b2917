"""Every launch plan of the wgmma tap-GEMM (csrc/conv_tc.cu) against fp64.

``tc_plan()`` picks the instantiation of a call - tile width BN 128 / 64 / 32, K-slab width SWB 128 / 64 bytes, the plain
or halo form, a K split with a fixed-order reduction - from the shape, the operand format, the partial-sum space and the
SM budget of the calling thread (``ops.launch_policy``).  One table of cases runs on all three operand formats at SM
budgets 1, 3, 16, 100 and the full device; every run logs the plan ``mtts_tc_plan_query`` reports for it and its error as
a fraction of the bar:
  * bf16x3 / f16x2: fp64 reference, fp32-grade bar 3e-5 * max(1, max|ref|);
  * f16: fp64 over the fp16-rounded operands, bar 1e-5 * max|ref| (only fp32 accumulation is left);
  * runs of one case and format whose plans are equal are bit-identical whatever the budget (each output element comes
    from one work item, or from a split reduction in a fixed order).
The CPU test at the end checks that the table, over the budgets, reaches every instantiation conv_tc() can launch and no
other, so a dispatcher change that orphans one fails without a GPU."""
import ctypes as C
import functools
import json
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from megatts2_b200 import _lib as L
from megatts2_b200 import pack

DEV = "cuda"
gpu = pytest.mark.gpu
FMTS = [L.TC_BF16X3, L.TC_F16X2, L.TC_F16]
FMT_NAMES = {L.TC_BF16X3: "bf16x3", L.TC_F16X2: "f16x2", L.TC_F16: "f16"}
BUDGETS = (1, 3, 16, 100, 0)          # SM budgets of the launching thread; 0 = the whole device
H100_SMS = 132                        # the full device in the host-only plan checks
NONE, RELU, LEAKY, TANH = L.ACT_NONE, L.ACT_RELU, L.ACT_LEAKY, L.ACT_TANH
PRE_SLOPE, POST_SLOPE, OP_SLOPE = 0.1, 0.2, 0.05


def _dense(M, K, N, **kw):
    return dict(kind="dense", B=1, T=M, Cin=K, Cout=N, k=1, dil=1, **kw)


def _conv(B, T, Cin, Cout, k, dil=1, **kw):
    return dict(kind="conv", B=B, T=T, Cin=Cin, Cout=Cout, k=k, dil=dil, **kw)


def _convt(B, T, Cin, Cout, s):
    """ConvTranspose1d(Cin, Cout, 2s, stride s, padding s/2) of the vocoder: a 2-tap conv with s * Cout columns over the
    leaky input, written at a negative output shift"""
    return dict(kind="convt", B=B, T=T, Cin=Cin, Cout=Cout, s=s, k=2, dil=1, pre=LEAKY, bias=True)


# name -> case.  Epilogue keys: bias, res, acc (accumulate into y), scale (out_scale), pre / post (activations), op (the
# operand-plane output for the next layer, with its own activation), partial (split-K partial-sum space).
CASES = {
    # dense layers: M tails (130, 1000), K tails (72: inside one 64-wide slab; 1000: 16 slabs, the last one partial)
    "dense_m130_k72_n192": _dense(130, 72, 192, bias=True, post=TANH, op=LEAKY),
    "dense_m1000_k1000_n1024": _dense(1000, 1000, 1024, bias=True, res=True, acc=True, scale=0.5),
    # Cin strictly between 32 and 64: 64-byte K-slabs, the K tail inside a slab, plain BN = 32
    "conv_cin48_cout32_k3": _conv(2, 700, 48, 32, 3, pad_mode=1, pre=LEAKY, bias=True, res=True),
    "conv_cin40_cout32_k5": _conv(3, 500, 40, 32, 5, post=LEAKY, bias=True, op=NONE),
    # C = 32, k = 3: halo 64 fills the 192-row halo buffer exactly; halo 66 falls back to the plain form
    "conv_c32_k3_dil32": _conv(2, 3000, 32, 32, 3, 32, pad_mode=1, pre=LEAKY, bias=True, res=True, acc=True, scale=1 / 3),
    "conv_c32_k3_dil33": _conv(2, 3000, 32, 32, 3, 33, pad_mode=1, pre=LEAKY, post=RELU, bias=True),
    # C = 64, k = 5 at B * ceil(T / 128) = 160 tiles (BN = 64 at every budget): halo 64 (halo form) and 68 (plain BN = 64)
    "conv_c64_k5_dil16": _conv(4, 5000, 64, 64, 5, 16, pad_mode=1, pre=LEAKY, bias=True, res=True),
    "conv_c64_k5_dil17": _conv(4, 5000, 64, 64, 5, 17, pad_mode=1, pre=LEAKY, bias=True, acc=True, scale=0.5, op=LEAKY),
    # C = 64 with an 18-row halo at 32 tiles: BN = 32 (plain) on the full device, the halo form under small budgets
    "conv_c64_k7_dil3": _conv(2, 2000, 64, 64, 7, 3, pad_mode=2, post=TANH, bias=True),
    # the four HiFi-GAN V1 up-samplers (s * Cout = 2048, 1024, 128, 64)
    "convt_up1": _convt(2, 100, 512, 256, 8),          # (the engine takes B * (T + 1) >= 128 rows)
    "convt_up2": _convt(2, 320, 256, 128, 8),
    "convt_up3": _convt(2, 2560, 128, 64, 2),
    "convt_up4": _convt(2, 5120, 64, 32, 2),
    # split-K dense layers (partial-sum space given): M tail, K tail, uneven slab splits, epilogues in the reduction
    "split_m130_k1000_n1024": _dense(130, 1000, 1024, bias=True, res=True, acc=True, scale=0.75, partial=True),
    "split_m130_k1000_n768": _dense(130, 1000, 768, bias=True, pre=LEAKY, post=RELU, op=RELU, partial=True),
    "split_m200_k4096_n512": _dense(200, 4096, 512, bias=True, post=LEAKY, partial=True),
    "split_m200_k4096_n384": _dense(200, 4096, 384, res=True, pre=RELU, op=NONE, partial=True),
}


# ------------------------------------------------------------------------------------------ plans (host only)
def _geometry(c):
    """(B, Tout, Cin, Cout, k, dil) of the tap-GEMM a case launches"""
    if c["kind"] == "convt":
        return c["B"], c["T"] + 1, c["Cin"], c["s"] * c["Cout"], 2, 1
    return c["B"], c["T"], c["Cin"], c["Cout"], c["k"], c["dil"]


def _partial_floats(c):
    return 8 * c["B"] * c["T"] * c["Cout"] if c.get("partial") else 0


def plan_of(c, fmt, sms):
    """The plan conv_tc() takes for case c on `sms` SMs.  The query has no out_shift argument, and conv_tc() keeps a
    transposed conv (out_shift set) off the halo form, so its queried plan is taken with halo = 0."""
    B, T, Cin, Cout, k, dil = _geometry(c)
    out = (C.c_int32 * 5)()
    L.check(L.lib().mtts_tc_plan_query(sms, B, T, Cin, Cout, k, dil, fmt, 4 * _partial_floats(c), 0, out))
    pl = dict(BN=out[0], splits=out[1], halo=out[3], swb=out[4])
    if c["kind"] == "convt":
        pl["halo"] = 0
    return pl


def instantiation(pl, fmt):
    """the conv_tc_kernel<BN, SWB, NP, HALO> a plan launches, with the split-K flag"""
    form = "halo" if pl["halo"] else ("split" if pl["splits"] > 1 else "plain")
    return form, pl["BN"], pl["swb"], 3 - fmt


# ------------------------------------------------------------------------------------------ inputs and references
def _gen(name):
    g = torch.Generator()
    g.manual_seed(zlib.crc32(name.encode()))
    return g


def _act(x, a, slope):
    return {NONE: lambda t: t, RELU: F.relu, LEAKY: lambda t: F.leaky_relu(t, slope), TANH: torch.tanh}[a](x)


@functools.lru_cache(maxsize=None)
def inputs(name):
    c = CASES[name]
    g = _gen(name)
    B, T, Cin, Cout, k = c["B"], c["T"], c["Cin"], c["Cout"], c["k"]
    x = torch.randn(B, T, Cin, generator=g) * 2
    if c["kind"] == "convt":
        w = torch.randn(Cin, Cout, 2 * c["s"], generator=g) / math.sqrt(2 * Cin)
    else:
        w = torch.randn(Cout, Cin, k, generator=g) / math.sqrt(Cin * k)
    d = dict(x=x, w=w, b=torch.randn(Cout, generator=g) if c.get("bias") else None)
    d["res"] = torch.randn(B, T, Cout, generator=g) if c.get("res") else None
    d["y0"] = torch.randn(B, T, Cout, generator=g) if c.get("acc") else None
    return d


def _pad(c):
    return 1 if c["kind"] == "convt" else c["dil"] * (c["k"] - 1) // 2


def padded_input(name):
    """the pre-activated input with its padding, (B, T + 2 pad, Cin) fp32: what the split writes as operand planes"""
    c = CASES[name]
    x = _act(inputs(name)["x"], c.get("pre", NONE), PRE_SLOPE).transpose(1, 2)
    pad, mode = _pad(c), c.get("pad_mode", 0)
    x = F.pad(x, (pad, pad), mode={1: "reflect", 2: "replicate"}[mode]) if mode else F.pad(x, (pad, pad))
    return x.transpose(1, 2).contiguous()


@functools.lru_cache(maxsize=None)
def reference(name, f16):
    """fp64 result of case `name`; f16: over the fp16-rounded operands the f16 engine multiplies"""
    c, d = CASES[name], inputs(name)
    q = (lambda t: t.half().double()) if f16 else (lambda t: t.double())
    b = d["b"].double() if d["b"] is not None else None
    xin = q(padded_input(name)).transpose(1, 2)
    if c["kind"] == "convt":
        s = c["s"]
        x = q(_act(d["x"], LEAKY, PRE_SLOPE)).transpose(1, 2)
        return F.conv_transpose1d(x, q(d["w"]), b, stride=s, padding=s // 2).transpose(1, 2)
    ref = F.conv1d(xin, q(d["w"]), b, dilation=c["dil"]).transpose(1, 2)
    ref = _act(ref, c.get("post", NONE), POST_SLOPE)
    if d["res"] is not None:
        ref = ref + d["res"].double()
    ref = ref * c.get("scale", 1.0)
    if d["y0"] is not None:
        ref = ref + d["y0"].double()
    return ref


def bar_of(ref, fmt):
    if fmt == L.TC_F16:
        return 1e-5 * ref.abs().max().item()
    return 3e-5 * max(1.0, ref.abs().max().item())


@functools.lru_cache(maxsize=None)
def _input_plane0(name, fmt):
    c = CASES[name]
    xp = padded_input(name)
    return pack.pack_tc_planes(xp.reshape(-1, c["Cin"]), fmt)[0].view(torch.int16).reshape(-1)


# ------------------------------------------------------------------------------------------ one launch
@functools.lru_cache(maxsize=None)
def _device_weights(name, fmt):
    c, d = CASES[name], inputs(name)
    if c["kind"] == "convt":
        wp, bp = pack.pack_conv_transpose(d["w"], d["b"], c["s"])
        return wp.to(DEV), bp.to(DEV), pack.pack_conv_transpose_tc_planes(wp.to(DEV), fmt)
    w32 = pack.pack_conv(d["w"]).to(DEV)
    b = d["b"].to(DEV) if d["b"] is not None else None
    return w32, b, pack.pack_conv_tc_planes(d["w"].to(DEV), fmt)


def launch(name, fmt, budget):
    """One tap-GEMM call of case `name` on the tensor-core engine under an SM budget -> (y, out planes | None, plane 0 of
    the activation split) on the host."""
    from megatts2_b200 import ops
    c, d = CASES[name], inputs(name)
    B, Tout, Cin, Cout, k, dil = _geometry(c)
    T = c["T"]
    w32, bias, planes = _device_weights(name, fmt)
    x = d["x"].to(DEV)
    p = L.ConvParams()
    p.x, p.x_batch_stride, p.ldx = x.data_ptr(), T * Cin, Cin
    p.w, p.bias = w32.data_ptr(), bias.data_ptr() if bias is not None else None
    p.B, p.Tin, p.Tout, p.Cin, p.Cout = B, T, Tout, Cin, Cout
    p.k, p.stride, p.dil, p.pad, p.pad_mode = k, 1, dil, _pad(c), c.get("pad_mode", 0)
    p.pre_act, p.pre_slope = c.get("pre", NONE), PRE_SLOPE
    p.post_act, p.post_slope = c.get("post", NONE), POST_SLOPE
    p.out_scale, p.accumulate = c.get("scale", 1.0), int(bool(c.get("acc")))
    keep = [x, w32, bias, planes]
    if c["kind"] == "convt":
        s, co = c["s"], c["Cout"]
        y = torch.empty(B, s * T, co, device=DEV)
        p.y_batch_stride, p.ldy = s * T * co, s * co
        p.out_shift, p.y_batch_elems = -(s // 2) * co, s * T * co
    else:
        y = d["y0"].to(DEV) if d["y0"] is not None else torch.empty(B, T, Cout, device=DEV)
        p.y_batch_stride, p.ldy = T * Cout, Cout
    p.y = y.data_ptr()
    if d["res"] is not None:
        r = d["res"].to(DEV)
        keep.append(r)
        p.res, p.res_batch_stride, p.ldr = r.data_ptr(), T * Cout, Cout
    rows = B * (Tout + dil * (k - 1))
    nbytes = 6 * rows * Cin + 4096
    scratch = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    p.w_tc, p.tc_scratch, p.tc_scratch_bytes, p.tc_fmt = planes.data_ptr(), scratch.data_ptr(), nbytes, fmt
    if c.get("partial"):
        part = torch.empty(_partial_floats(c), dtype=torch.float32, device=DEV)
        keep.append(part)
        p.tc_partial, p.tc_partial_bytes = part.data_ptr(), part.numel() * 4
    op = None
    if "op" in c:
        op = torch.full((3 - fmt, B, T, Cout), 7.0, dtype=pack.plane_dtype(fmt), device=DEV)
        p.tc_out_planes, p.tc_out_plane_stride, p.tc_out_ld = op.data_ptr(), B * T * Cout, Cout
        p.tc_out_tp, p.tc_out_hl, p.tc_out_act, p.tc_out_slope = T, 0, c["op"], OP_SLOPE
    ops.tc_overflow_bind(torch.device(DEV))
    with ops.launch_policy(budget):
        L.check(L.lib().mtts_conv1d_f32(C.byref(p), ops._stream()))
    torch.cuda.synchronize()
    del keep
    off = (-scratch.data_ptr()) % 1024
    n = B * (Tout + dil * (k - 1)) * Cin
    plane0 = scratch[off:off + 2 * n].view(torch.int16).cpu()
    return y.cpu(), op.cpu() if op is not None else None, plane0


def run_case(name, fmt, budgets=BUDGETS):
    """Runs case `name` in format `fmt` at every budget; checks each run against fp64 and equal plans for bit identity.
    Returns one record per run: budget, SMs, plan, error / bar."""
    from megatts2_b200 import ops
    c = CASES[name]
    ref = reference(name, fmt == L.TC_F16)
    bar = bar_of(ref, fmt)
    full = ops.sm_count(torch.device(DEV))
    seen, records = {}, []
    for budget in budgets:
        sms = budget if 0 < budget < full else full
        pl = plan_of(c, fmt, sms)
        y, op, plane0 = launch(name, fmt, budget)
        # the tensor-core engine ran: its activation split is in the scratch (an FFMA fall-back leaves no operand planes)
        assert torch.equal(plane0, _input_plane0(name, fmt)), f"{name} {FMT_NAMES[fmt]} @{sms}: no operand planes"
        err = (y.double() - ref).abs().max().item()
        rec = dict(case=name, fmt=FMT_NAMES[fmt], budget=budget, sms=sms, plan=pl, err=err, bar=bar)
        records.append(rec)
        print(f"{name:28s} {FMT_NAMES[fmt]:6s} sms {sms:3d}  {instantiation(pl, fmt)} splits {pl['splits']}  "
              f"err {err:.3e} = {err / bar:.3f} of the bar")
        assert err <= bar, rec
        if op is not None:
            spec = pack.pack_tc_planes(_act(y, c["op"], OP_SLOPE).reshape(-1, c["Cout"]), fmt)
            assert torch.equal(op.view(torch.int16).reshape(spec.shape), spec.view(torch.int16)), f"{rec}: operand planes"
        key = json.dumps(pl, sort_keys=True)
        if key in seen:
            assert torch.equal(y, seen[key]), f"{rec}: not bit-identical to an earlier run of the same plan"
        else:
            seen[key] = y
    return records


# ------------------------------------------------------------------------------------------ GPU: the table
@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("fmt", FMTS, ids=FMT_NAMES.get)
@pytest.mark.parametrize("name", list(CASES))
def test_tap_gemm_plans_vs_fp64(name, fmt):
    import helpers
    for rec in run_case(name, fmt):
        helpers.record("tc_plans", rec)


ENCODER_SHAPE = (2, 100)             # M = 200 rows: the out-projection and FF2 split K, their reductions carry a LayerNorm
ENCODER_BARS = {L.TC_BF16X3: 2e-4, L.TC_F16X2: 2e-4, L.TC_F16: 2e-2}   # the bars of the encoder tests on each engine


def _random_encoder(D, H, seed):
    from megatts2_b200.modules.transformer import TransformerEncoder, TransformerEncoderLayer
    enc = TransformerEncoder(TransformerEncoderLayer(dim=D, ff_dim=4 * D, conv_ff=False, n_heads=H), 2)
    g = torch.Generator()
    g.manual_seed(seed)
    with torch.no_grad():
        for n, prm in enc.named_parameters():
            if prm.dim() == 2:
                prm.copy_(torch.randn(prm.shape, generator=g) / math.sqrt(prm.shape[1]))
            elif "norm" in n and n.endswith("weight"):
                prm.copy_(1 + 0.2 * torch.randn(prm.shape, generator=g))
            else:
                prm.copy_(0.2 * torch.randn(prm.shape, generator=g))
    return enc


@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("fmt", FMTS, ids=FMT_NAMES.get)
@pytest.mark.parametrize("D,H", [(384, 6), (512, 8)])
def test_splitk_layernorm_reduction_vs_fp64(D, H, fmt):
    """The split-K reductions that carry a LayerNorm (tc_splitk_reduce_ln_kernel<3 | 4>): a 2-layer linear-FF encoder at
    d_model 384 / 512, whose out-projection and FF2 split K with the next LayerNorm riding on the reduction (ops.conv1d
    passes no partial-sum space, so the encoder is the way in), against the oracle's encoder in fp64."""
    from oracle import ref_megatts2 as R
    B, T = ENCODER_SHAPE
    M = B * T
    out = (C.c_int32 * 5)()
    split = []
    for K in (D, 4 * D):               # out-projection (LN2 rides), FF2 (the next layer's LN1 rides)
        L.check(L.lib().mtts_tc_plan_query(H100_SMS, 1, M, K, D, 1, 1, fmt, 64 << 20, 1, out))
        split.append(out[1])
    print(f"encoder D {D} {FMT_NAMES[fmt]}: splits (out-proj, FF2) {split}")
    assert split[1] > 1
    enc = _random_encoder(D, H, D + fmt)
    x = torch.randn(B, T, D, generator=_gen(f"enc{D}"))
    sd = {k: v.double() for k, v in enc.state_dict().items()}
    ref = R.encoder(R.SD(sd), x.double(), 2, H, False)
    enc = enc.to(DEV).eval()
    enc.engine = {L.TC_BF16X3: pack.ENGINE_BF16X3, L.TC_F16X2: pack.ENGINE_F16X2, L.TC_F16: pack.ENGINE_F16}[fmt]
    y = enc(x.to(DEV))
    err = (y.cpu().double() - ref).abs().max().item()
    print(f"  err {err:.3e} = {err / ENCODER_BARS[fmt]:.3f} of the bar")
    assert err < ENCODER_BARS[fmt]
    assert torch.equal(y, enc(x.to(DEV))), "the split-K reduction order is fixed"


# ------------------------------------------------------------------------------------------ CPU: coverage of the table
def test_default_table_reaches_every_instantiation():
    """The plans of the table's cases, at budgets 1, 3, 16, 100 and 132 SMs, together launch every conv_tc_kernel
    instantiation conv_tc() has and no other, and no split plan runs at a tile width other than 128."""
    reached = set()
    for n in CASES:
        for fmt in FMTS:
            for sms in (1, 3, 16, 100, H100_SMS):
                pl = plan_of(CASES[n], fmt, sms)
                assert pl["splits"] == 1 or pl["BN"] == 128, (n, fmt, sms, pl)
                reached.add(instantiation(pl, fmt))
    want = {("plain", bn, 128, npl) for bn in (128, 64, 32) for npl in (1, 2, 3)}
    want |= {("plain", 32, 64, npl) for npl in (1, 2, 3)}
    want |= {("halo", bn, swb, npl) for bn, swb in ((32, 64), (64, 128)) for npl in (1, 2, 3)}
    want |= {("split", 128, 128, npl) for npl in (1, 2, 3)}
    assert not want - reached, sorted(want - reached)
    assert not reached - want, sorted(reached - want)       # a plan outside the instantiations conv_tc() can launch
