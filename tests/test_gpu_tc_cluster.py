"""2-CTA clusters on the wgmma tap-GEMM (csrc/conv_tc.cu, CL = 2): the two CTAs of a cluster share the weight tile of a
pair item through TMA multicast, each computes its own row tile.

Each output row is computed by the same MMAs in the same k order and the same epilogue whether its row tile runs in a
cluster or alone, so a clustered launch must equal, bit for bit, the same launch on single CTAs (``ops.launch_policy(...,
pairs=False)``), and both must meet the fp64 bars of test_gpu_tc_plans.py.  The cases cover tile widths BN 128 / 64 / 32
(128- and 64-byte K-slabs), odd row-tile counts (the rank-1 CTA of the last pair runs a dummy item), pairs that straddle
two batch items, the transposed-conv output shift and every epilogue key, at SM budgets of 2, 3 and 4 (one or two
clusters walk dozens of pair items, so the stage ring and its phases wrap many times) and on the whole device.  The CPU
tests pin the cluster rule of the launch plan."""
import ctypes as C
import functools
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

import helpers
from megatts2_b200 import _lib as L
from megatts2_b200 import pack

DEV = "cuda"
gpu = pytest.mark.gpu
FMTS = [L.TC_BF16X3, L.TC_F16X2, L.TC_F16]
FMT_NAMES = {L.TC_BF16X3: "bf16x3", L.TC_F16X2: "f16x2", L.TC_F16: "f16"}
BUDGETS = (2, 3, 4, 0)                # SM budgets of the launching thread; 0 = the whole device
H100_SMS = 132
NONE, RELU, LEAKY, TANH = L.ACT_NONE, L.ACT_RELU, L.ACT_LEAKY, L.ACT_TANH
PRE_SLOPE, POST_SLOPE, OP_SLOPE = 0.1, 0.2, 0.05


def _conv(B, T, Cin, Cout, k, dil=1, **kw):
    return dict(kind="conv", B=B, T=T, Cin=Cin, Cout=Cout, k=k, dil=dil, **kw)


# name -> case; row tiles = B * ceil(Tout / ROWS), ROWS = 64 at BN = 128, else 128 (the plan's BN at budgets 2 ... 4)
CASES = {
    # dense, BN 128: 17 row tiles (odd), M and K tails
    "dense_m1030_k200_n256": _conv(1, 1030, 200, 256, 1, bias=True, post=TANH, op=LEAKY),
    # k = 1 over 3 batch items, BN 128: 5 row tiles each, so pairs (4, 0) and (4, 0) straddle batch items; 15 in all
    "dense_b3_t300_k128_n384": _conv(3, 300, 128, 384, 1, bias=True, res=True, acc=True, scale=0.5),
    # conv, BN 64 (Cout = 64, Cin = 128: plain form): 3 x 5 row tiles, straddling pairs, reflect padding
    "conv_b3_t520_c128_n64_k3": _conv(3, 520, 128, 64, 3, 2, pad_mode=1, pre=LEAKY, bias=True, res=True),
    # conv, BN 32 on 128-byte K-slabs: 2 x 8 row tiles (even)
    "conv_b2_t900_c128_n32_k5": _conv(2, 900, 128, 32, 5, post=RELU, bias=True, acc=True, scale=0.75, op=NONE),
    # conv, BN 32 on 64-byte K-slabs (Cin 48): 3 x 3 row tiles, replicate padding
    "conv_b3_t300_c48_n32_k3": _conv(3, 300, 48, 32, 3, pad_mode=2, pre=LEAKY, bias=True, res=True),
    # ConvTranspose1d(256, 128, 16, stride 8, padding 4) = a 2-tap conv of 1024 columns at a negative output shift:
    # 3 x ceil(131 / 64) = 9 row tiles at BN 128
    "convt_b3_t130_s8": dict(kind="convt", B=3, T=130, Cin=256, Cout=128, s=8, k=2, dil=1, pre=LEAKY, bias=True),
}


def _geometry(c):
    if c["kind"] == "convt":
        return c["B"], c["T"] + 1, c["Cin"], c["s"] * c["Cout"], 2, 1
    return c["B"], c["T"], c["Cin"], c["Cout"], c["k"], c["dil"]


def plan_ex(sms, B, T, Cin, Cout, k=1, dil=1, fmt=L.TC_F16X2, partial=0, ln=0, pairs=1):
    out = (C.c_int32 * 7)()
    L.check(L.lib().mtts_tc_plan_query_ex(sms, B, T, Cin, Cout, k, dil, fmt, partial, ln, pairs, out))
    return dict(BN=out[0], splits=out[1], pair=out[2], halo=out[3], swb=out[4], cluster=out[5], ctas=out[6])


def row_tiles(B, T, BN):
    return B * -(-T // (64 if BN == 128 else 128))


# ------------------------------------------------------------------------------------------ CPU: the cluster rule
def test_cluster_rule_of_the_launch_plan():
    """2-CTA clusters for the plain form without a K split and with at least two row tiles, at every tile width; single
    CTAs for split-K launches, the halo form, one row tile, budgets below 2 SMs and pairs=False.  A clustered grid is
    even: an odd budget leaves one SM unused."""
    cd = lambda a, b: -(-a // b)
    # split K (early AR steps): single CTAs
    pl = plan_ex(H100_SMS, 1, 64 * 4, 4096, 1024, partial=64 << 20, ln=1)
    assert pl["splits"] > 1 and pl["cluster"] == 1
    # halo form (C = 32 / 64 vocoder convs): single CTAs
    for Cin, swb in ((32, 64), (64, 128)):
        pl = plan_ex(H100_SMS, 64, 66816 // (Cin // 32), Cin, Cin, k=7, dil=3)
        assert pl["halo"] == 1 and pl["swb"] == swb and pl["cluster"] == 1, pl
    # one row tile: 64 rows at BN 128, 128 rows at BN 64 / 32
    assert plan_ex(H100_SMS, 1, 64, 1024, 1024)["cluster"] == 1
    assert plan_ex(H100_SMS, 1, 128, 1024, 64)["cluster"] == 1
    assert plan_ex(H100_SMS, 1, 128, 1024, 32)["cluster"] == 1
    # odd and even row-tile counts at every tile width: clusters; the grid covers the pair items or the even budget
    for N in (1024, 64, 32):
        for M in (1024, 1030, 5888, 129, 65):
            pl = plan_ex(H100_SMS, 1, M, 1024, N)
            rt = row_tiles(1, M, pl["BN"])
            if rt < 2:
                assert pl["cluster"] == 1
                continue
            assert pl["cluster"] == 2 and pl["splits"] == 1 and pl["halo"] == 0, (M, N, pl)
            assert pl["ctas"] == 2 * min(cd(rt, 2) * cd(N, pl["BN"]), H100_SMS // 2), (M, N, pl)
    # plain-form convolutions at C = 128 / 256 (and k = 1 over several batch items)
    assert plan_ex(H100_SMS, 64, 8352, 128, 128, k=7, dil=3)["cluster"] == 2
    assert plan_ex(H100_SMS, 64, 4176, 256, 256, k=7, dil=3)["cluster"] == 2
    # odd SM budgets round down to an even grid; below 2 SMs single CTAs
    for sms in (3, 5, 7, 131):
        pl = plan_ex(sms, 1, 5888, 1024, 3072)
        assert pl["cluster"] == 2 and pl["ctas"] == sms - 1, (sms, pl)
    pl = plan_ex(1, 1, 5888, 1024, 3072)
    assert pl["cluster"] == 1 and pl["ctas"] == 1
    # pairs = 0 (ops.launch_policy(..., pairs=False)): single CTAs, the same tile plan otherwise
    for sms in (2, 66, H100_SMS):
        on, off = plan_ex(sms, 1, 5888, 1024, 3072), plan_ex(sms, 1, 5888, 1024, 3072, pairs=0)
        assert off["cluster"] == 1 and off["ctas"] == min(row_tiles(1, 5888, off["BN"]) * cd(3072, off["BN"]), sms)
        assert {k: v for k, v in on.items() if k not in ("cluster", "ctas")} == \
               {k: v for k, v in off.items() if k not in ("cluster", "ctas")}
    # the five-field query is the extended one with clusters allowed; its CTA-pair field stays 0
    out5 = (C.c_int32 * 5)()
    L.check(L.lib().mtts_tc_plan_query(H100_SMS, 1, 5888, 1024, 3072, 1, 1, L.TC_F16X2, 0, 0, out5))
    pl = plan_ex(H100_SMS, 1, 5888, 1024, 3072)
    assert list(out5) == [pl["BN"], pl["splits"], 0, pl["halo"], pl["swb"]]


def test_cluster_cases_reach_every_clustered_instantiation():
    """The cases below, at budgets 2 ... 4, launch every clustered instantiation (BN 128 / 64 / 32 on 128-byte K-slabs,
    BN 32 on 64-byte K-slabs, each operand format) with an odd and an even row-tile count among them."""
    reached, parity = set(), set()
    for name, c in CASES.items():
        B, T, Cin, Cout, k, dil = _geometry(c)
        for fmt in FMTS:
            for sms in (2, 3, 4):
                pl = plan_ex(sms, B, T, Cin, Cout, k, dil, fmt)
                assert pl["cluster"] == 2 and pl["halo"] == 0 and pl["ctas"] == 2 * (sms // 2), (name, sms, pl)
                reached.add((pl["BN"], pl["swb"], 3 - fmt))
                parity.add(row_tiles(B, T, pl["BN"]) % 2)
    want = {(bn, 128, npl) for bn in (128, 64, 32) for npl in (1, 2, 3)} | {(32, 64, npl) for npl in (1, 2, 3)}
    assert reached == want, sorted(want ^ reached)
    assert parity == {0, 1}


# ------------------------------------------------------------------------------------------ GPU
def _gen(name):
    g = torch.Generator()
    g.manual_seed(zlib.crc32(name.encode()))
    return g


def _act(x, a, slope):
    return {NONE: lambda t: t, RELU: F.relu, LEAKY: lambda t: F.leaky_relu(t, slope), TANH: torch.tanh}[a](x)


@functools.lru_cache(maxsize=None)
def inputs(name):
    c, g = CASES[name], _gen(name)
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


@functools.lru_cache(maxsize=None)
def reference(name, f16):
    """fp64 result; f16: over the fp16-rounded operands the f16 engine multiplies"""
    c, d = CASES[name], inputs(name)
    q = (lambda t: t.half().double()) if f16 else (lambda t: t.double())
    b = d["b"].double() if d["b"] is not None else None
    x = _act(d["x"], c.get("pre", NONE), PRE_SLOPE)
    if c["kind"] == "convt":
        s = c["s"]
        return F.conv_transpose1d(q(x).transpose(1, 2), q(d["w"]), b, stride=s, padding=s // 2).transpose(1, 2)
    pad, mode = _pad(c), c.get("pad_mode", 0)
    x = x.transpose(1, 2)
    x = F.pad(x, (pad, pad), mode={1: "reflect", 2: "replicate"}[mode]) if mode else F.pad(x, (pad, pad))
    ref = F.conv1d(q(x), q(d["w"]), b, dilation=c["dil"]).transpose(1, 2)
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
def _device_weights(name, fmt):
    c, d = CASES[name], inputs(name)
    if c["kind"] == "convt":
        wp, bp = pack.pack_conv_transpose(d["w"], d["b"], c["s"])
        return wp.to(DEV), bp.to(DEV), pack.pack_conv_transpose_tc_planes(wp.to(DEV), fmt)
    b = d["b"].to(DEV) if d["b"] is not None else None
    return pack.pack_conv(d["w"]).to(DEV), b, pack.pack_conv_tc_planes(d["w"].to(DEV), fmt)


def launch(name, fmt, budget, pairs):
    """One tap-GEMM call of case `name` on the tensor-core engine -> (y, operand-plane output | None) on the host"""
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
        y = torch.full((B, s * T, co), 5.0, device=DEV)
        p.y_batch_stride, p.ldy = s * T * co, s * co
        p.out_shift, p.y_batch_elems = -(s // 2) * co, s * T * co
    else:
        y = d["y0"].to(DEV) if d["y0"] is not None else torch.full((B, T, Cout), 5.0, device=DEV)
        p.y_batch_stride, p.ldy = T * Cout, Cout
    p.y = y.data_ptr()
    if d["res"] is not None:
        r = d["res"].to(DEV)
        keep.append(r)
        p.res, p.res_batch_stride, p.ldr = r.data_ptr(), T * Cout, Cout
    nbytes = 6 * B * (Tout + dil * (k - 1)) * Cin + 4096
    scratch = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    p.w_tc, p.tc_scratch, p.tc_scratch_bytes, p.tc_fmt = planes.data_ptr(), scratch.data_ptr(), nbytes, fmt
    op = None
    if "op" in c:
        op = torch.full((3 - fmt, B, T, Cout), 7.0, dtype=pack.plane_dtype(fmt), device=DEV)
        p.tc_out_planes, p.tc_out_plane_stride, p.tc_out_ld = op.data_ptr(), B * T * Cout, Cout
        p.tc_out_tp, p.tc_out_hl, p.tc_out_act, p.tc_out_slope = T, 0, c["op"], OP_SLOPE
    ops.tc_overflow_bind(torch.device(DEV))
    with ops.launch_policy(budget, pairs=pairs):
        L.check(L.lib().mtts_conv1d_f32(C.byref(p), ops._stream()))
    torch.cuda.synchronize()
    del keep
    return y.cpu(), op.cpu() if op is not None else None


@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("fmt", FMTS, ids=FMT_NAMES.get)
@pytest.mark.parametrize("name", list(CASES))
def test_clustered_launch_equals_single_cta_launch(name, fmt):
    from megatts2_b200 import ops
    c = CASES[name]
    B, Tout, Cin, Cout, k, dil = _geometry(c)
    ref = reference(name, fmt == L.TC_F16)
    bar = bar_of(ref, fmt)
    full = ops.sm_count(torch.device(DEV))
    for budget in BUDGETS:
        sms = budget if 0 < budget < full else full
        pl = plan_ex(sms, B, Tout, Cin, Cout, k, dil, fmt)
        assert pl["cluster"] == 2, pl
        y2, op2 = launch(name, fmt, budget, pairs=True)
        y1, op1 = launch(name, fmt, budget, pairs=False)
        err = (y2.double() - ref).abs().max().item()
        rec = dict(case=name, fmt=FMT_NAMES[fmt], sms=sms, BN=pl["BN"], swb=pl["swb"], ctas=pl["ctas"], err=err, bar=bar)
        helpers.record("tc_cluster", rec)
        print(f"{name:26s} {FMT_NAMES[fmt]:6s} sms {sms:3d} BN {pl['BN']:3d} swb {pl['swb']:3d} "
              f"row tiles {row_tiles(B, Tout, pl['BN']):3d}  err {err:.3e} = {err / bar:.3f} of the bar")
        assert err <= bar, rec
        assert torch.equal(y2, y1), f"{rec}: clustered != single-CTA"
        if op2 is not None:
            assert torch.equal(op2.view(torch.int16), op1.view(torch.int16)), f"{rec}: operand planes"
            spec = pack.pack_tc_planes(_act(y2, c["op"], OP_SLOPE).reshape(-1, c["Cout"]), fmt)
            assert torch.equal(op2.view(torch.int16).reshape(spec.shape), spec.view(torch.int16)), f"{rec}: operand planes"


@gpu
@pytest.mark.timeout(600)
def test_graph_replay_of_clustered_decodes_matches_single_cta_eager(weights_cpu):
    """The AR decodes replayed from CUDA graphs, whose dense layers run as 2-CTA cluster launches with programmatic
    dependent launch edges, give the ids / durations of an eager enqueue on single CTAs bit for bit."""
    from megatts2_b200 import graphs, ops
    plm = helpers.build_plm(weights_cpu("plm"), DEV)
    adm = helpers.build_adm(weights_cpu("adm"), DEV)
    g = _gen("graph")
    tc8 = F.relu(torch.randn(16, 12, 512, generator=g)).to(DEV)
    tc8b = F.relu(torch.randn(16, 12, 512, generator=g)).to(DEV)
    with graphs.disabled(), ops.launch_policy(0, pairs=False):
        ref_a, ref_b = plm.infer(tc8), plm.infer(tc8b)
        dref_a, dref_b = adm.infer(tc8, return_raw=True), adm.infer(tc8b, return_raw=True)
    plm._graphs().clear(); adm._graphs().clear()
    outs = [plm.infer(tc8), plm.infer(tc8), plm.infer(tc8b), plm.infer(tc8)]          # eager, capture + replay, replays
    assert all(torch.equal(o, r) for o, r in zip(outs, (ref_a, ref_a, ref_b, ref_a)))
    douts = [adm.infer(tc8, return_raw=True), adm.infer(tc8, return_raw=True), adm.infer(tc8b, return_raw=True)]
    for (d, r), (dr, rr) in zip(douts, (dref_a, dref_a, dref_b)):
        assert torch.equal(d, dr) and torch.equal(r, rr)
