"""The tensor-core engines across the fp32 range, and the default formats' plane writers bit for bit.

The split operand formats are fp32-grade in significance, but their planes have their own exponent ranges:
  bf16x3: x = p1 + p2 + p3 (bf16) has the fp32 range, |x - x^| <= 2^-22 |x| at every normal magnitude;
  f16x2 : x = p1 + p2' * 2^-11 (fp16) has |x - x^| <= 2^-22 |x| + 2^-36 below 65504 (p1 is subnormal below 2^-14 and
          both planes vanish below about 2^-35), and poisons + flags anything above 65504.
These tests pin both edges: the representation bounds, exact scale equivariance on bf16x3, the documented lower edge on
f16x2, training gradients that span the fp32 range (they run on bf16x3), and attention inputs above the fp16 range under
the engines that promise the fp32 range (bf16x3, FFMA).  Every reference is fp64 on the CPU over the exact fp32 inputs
the kernel received; the plane writers are specified by ``pack.pack_tc_planes`` on the CPU applied to the fp32 values
the same launch stored."""
import ctypes as C
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import helpers
from megatts2_b200 import _lib as L
from megatts2_b200 import pack

DEV = "cuda"
gpu = pytest.mark.gpu
TIMEOUT = pytest.mark.timeout(600)
FMTS = [pack.FMT_BF16X3, pack.FMT_F16X2, pack.FMT_F16]
FMT_NAMES = {pack.FMT_BF16X3: "bf16x3", pack.FMT_F16X2: "f16x2", pack.FMT_F16: "f16"}
DEFAULT_FMTS = [pack.FMT_BF16X3, pack.FMT_F16X2]


def gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


def _bits(t):
    return t.contiguous().view(torch.int16).cpu()


def _value(planes, fmt):
    """fp64 value the planes represent"""
    p = planes.double()
    if fmt == pack.FMT_F16X2:
        return p[0] + p[1] * 2.0 ** -11
    return p.sum(0)


# ------------------------------------------------------------------------------------------ range of the split
def _sweep():
    """(77, 36) fp32: row e < 76 holds 2^(e-60) * m for 32 random mantissas m in [1, 2) with random signs, then
    +-2^(e-60) and +-1.5 * 2^(e-60) exactly; the last row values around and far above the fp16 ceiling"""
    g = gen(71)
    rows = []
    for e in range(-60, 16):
        m = 1 + torch.rand(32, generator=g, dtype=torch.float64)
        s = torch.where(torch.rand(32, generator=g) < 0.5, -1.0, 1.0).double()
        exact = torch.tensor([1.0, -1.0, 1.5, -1.5], dtype=torch.float64)
        rows.append(torch.cat([m * s, exact]) * 2.0 ** e)
    above = torch.tensor([65505.0, 65519.0, 65520.0, 65536.0, 7e4, 1e6, 1e12, 1e30, 3e38], dtype=torch.float64)
    rows.append(torch.cat([above, -above, above[:9] * 0.75, -above[:9] * 0.5]))
    return torch.stack(rows).float()


def test_split_representation_bounds_across_the_fp32_range():
    x = _sweep()
    ax = x.double().abs()
    xh = _value(pack.pack_tc_planes(x, pack.FMT_BF16X3), pack.FMT_BF16X3)
    assert bool(((x.double() - xh).abs() <= 2.0 ** -22 * ax).all()), "bf16x3 keeps 22 bits at every magnitude"
    p = pack.pack_tc_planes(x, pack.FMT_F16X2)
    inr = ax <= 65504
    xh = _value(p, pack.FMT_F16X2)
    err = (x.double() - xh).abs()
    assert bool((err[inr] <= 2.0 ** -22 * ax[inr] + 2.0 ** -36).all()), "f16x2 lower edge"
    # the absolute term is real: far below 2^-14 the relative error is large, below ~2^-36 the value is gone
    tiny = ax < 2.0 ** -37
    assert bool((xh[tiny] == 0).all())
    # above the range: the value is poisoned (p1 = +-inf from 65520 on) - the device split also raises the flag
    big = ax >= 65520
    assert big.any() and not bool(torch.isfinite(xh[big]).any())


@gpu
@TIMEOUT
def test_split_device_matches_host_bit_for_bit_and_flags_the_ceiling():
    from megatts2_b200 import ops
    dev = torch.device(DEV)
    ops.tc_overflow_bind(dev)
    x = _sweep()
    inr = x.abs() <= 65504
    xin = torch.where(inr, x, torch.zeros_like(x))
    for fmt in FMTS:
        ops.tc_overflow(dev)
        host, d = pack.pack_tc_planes(xin, fmt), pack.pack_tc_planes(xin.to(DEV), fmt)
        assert host.dtype == d.dtype and host.shape == d.shape
        assert torch.equal(_bits(host), _bits(d)), FMT_NAMES[fmt]
        assert not ops.tc_overflow(dev), FMT_NAMES[fmt]
        host, d = pack.pack_tc_planes(x, fmt), pack.pack_tc_planes(x.to(DEV), fmt)
        assert torch.equal(_bits(host), _bits(d)), FMT_NAMES[fmt]
        assert ops.tc_overflow(dev) == (fmt != pack.FMT_BF16X3), FMT_NAMES[fmt]


# ------------------------------------------------------------------------------------------ tap-GEMM scale equivariance
TAP_CASES = [
    dict(kind="linear", M=256, K=1024, N=256),
    dict(kind="conv", B=2, T=300, Cin=64, Cout=64, k=7, dil=3, pad_mode=0),          # halo form
    dict(kind="conv", B=2, T=200, Cin=256, Cout=256, k=3, dil=1, pad_mode=1),        # reflect, BN 128
]


def _ids(c):
    return "-".join(f"{k}{v}" for k, v in c.items())


def _tap_inputs(c, bounded):
    """x and w at O(1) / O(1/32); ``bounded`` keeps every |value| in [0.5, 2] (resp. /32) so that no product of planes
    leaves the fp32 normal range at the extreme scales of the bf16x3 sweep"""
    g = gen(sum(v for v in c.values() if isinstance(v, int)))
    xs = (c["M"], c["K"]) if c["kind"] == "linear" else (c["B"], c["T"], c["Cin"])
    ws = (c["N"], c["K"]) if c["kind"] == "linear" else (c["Cout"], c["Cin"], c["k"])

    def draw(shape):
        if not bounded:
            return torch.randn(shape, generator=g)
        sgn = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
        return sgn * (0.5 + 1.5 * torch.rand(shape, generator=g))
    return draw(xs), draw(ws) / 32


def _tap_run(c, x, w, fmt):
    from megatts2_b200 import ops
    if c["kind"] == "linear":
        return ops.linear_tc(x.to(DEV), pack.pack_tc_planes(w.to(DEV), fmt)).cpu()
    k, dil = c["k"], c["dil"]
    y = ops.conv1d(x.to(DEV), pack.pack_conv(w).to(DEV), k=k, dil=dil, pad=dil * (k - 1) // 2, pad_mode=c["pad_mode"],
                   pre_act=L.ACT_LEAKY, pre_slope=0.1, w_tc=pack.pack_conv_tc_planes(w.to(DEV), fmt))
    return y.cpu()


def _tap_ref(c, x, w):
    """fp64 result, sum |x||w| and sum (|x| + |w|) per output element (x after the pre-activation)"""
    if c["kind"] == "linear":
        x64, w64 = x.double(), w.double()
        return x64 @ w64.t(), x64.abs() @ w64.abs().t(), x64.abs().sum(1, keepdim=True) + w64.abs().sum(1)
    k, dil, pm = c["k"], c["dil"], c["pad_mode"]
    pad = dil * (k - 1) // 2
    xt = F.leaky_relu(x, 0.1).double().transpose(1, 2)
    xt = F.pad(xt, (pad, pad), mode="reflect") if pm == 1 else F.pad(xt, (pad, pad))
    w64 = w.double()

    def conv(a, b):
        return F.conv1d(a, b, dilation=dil).transpose(1, 2)
    return conv(xt, w64), conv(xt.abs(), w64.abs()), conv(xt.abs(), torch.ones_like(w64)) + w64.abs().sum((1, 2))


@gpu
@TIMEOUT
@pytest.mark.parametrize("c", TAP_CASES, ids=_ids)
def test_tap_gemm_bf16x3_is_scale_equivariant_bit_for_bit(c):
    """Every bf16 plane of x * 2^s is 2^s times a plane of x and stays normal, and fp32 products scale exactly: any
    difference from 2^s * y(x) is a kernel bug (a plane read at the wrong scale, a flushed or dropped term)."""
    x, w = _tap_inputs(c, bounded=True)
    y0 = _tap_run(c, x, w, pack.FMT_BF16X3)
    ref, s_xw, _ = _tap_ref(c, x, w)
    assert bool(((y0.double() - ref).abs() <= 3e-5 * s_xw).all())
    for s in (-60, -40, -20, 20, 40):
        f = 2.0 ** s
        assert torch.equal(_tap_run(c, x * f, w, pack.FMT_BF16X3), y0 * f), f"x * 2^{s}"
        assert torch.equal(_tap_run(c, x, w * f, pack.FMT_BF16X3), y0 * f), f"w * 2^{s}"


@gpu
@TIMEOUT
@pytest.mark.parametrize("c", TAP_CASES, ids=_ids)
def test_tap_gemm_f16x2_error_across_scales(c):
    """fp32-grade for s in [-8, 8]; below that the documented lower edge, derived from the per-operand bound
    |x - x^| <= 2^-22 |x| + 2^-36:  4 (2^-21 sum|x||w| + 2^-36 sum(|x| + |w|)) + 3e-5 sum|x||w|."""
    x, w = _tap_inputs(c, bounded=False)
    for s in (-40, -28, -20, -14, -8, -4, 0, 4, 8):
        xs = x * 2.0 ** s
        ref, s_xw, s_sum = _tap_ref(c, xs, w)
        err = (_tap_run(c, xs, w, pack.FMT_F16X2).double() - ref).abs()
        bar = 3e-5 * s_xw
        if s < -8:
            bar = bar + 4 * (2.0 ** -21 * s_xw + 2.0 ** -36 * s_sum)
        worst = (err / bar).max().item()
        print(f"f16x2 s = {s:4d}: worst error / bar {worst:.3e}")
        assert worst <= 1.0, (s, worst)


# ------------------------------------------------------------------------------------------ training products
def _softmax_grad(x, w, ramp, seed):
    """dY = softmax(x W^T + bias) - onehot, fp32; bias ramps from 0 down to -ramp over the codes (the tail is a band the
    model has learnt to rule out: p down to e^-ramp), targets drawn from the plausible first quarter"""
    V = w.shape[0]
    logits = x @ w.t() + torch.linspace(0, -ramp, V)
    t = torch.randint(0, max(1, V // 4), (x.shape[0],), generator=gen(seed))
    return torch.softmax(logits, -1) - F.one_hot(t, V).float()


def _linear_grads(x, w, dy):
    from megatts2_b200 import autograd as A
    xd = x.to(DEV).requires_grad_(True)
    wd = w.to(DEV).requires_grad_(True)
    A.linear(xd, wd).backward(dy.to(DEV))
    return xd.grad.cpu(), wd.grad.cpu()


def _row_rel_l2(got, ref):
    n = ref.norm(dim=1)
    keep = n > 0
    return ((got.double() - ref).norm(dim=1)[keep] / n[keep])


@gpu
@TIMEOUT
@pytest.mark.parametrize("engine", [pack.ENGINE_F16X2, pack.ENGINE_BF16X3, pack.ENGINE_F16], ids=["f16x2", "bf16x3", "f16"])
def test_predict_layer_gradients_fp32_grade_per_row(engine):
    """The PLM predict layer's gradients, dW = dY^T X and dX = dY W with dY = softmax - onehot: the rows of codes the model
    rules out carry gradients of e^-40 scale, which an fp16 plane flushes to zero.  Each row is held to fp64 on its own
    (a whole-tensor norm is dominated by the large rows)."""
    g = gen(41)
    V, K, M = 1024, 1024, 256
    x = torch.randn(M, K, generator=g)
    w = torch.randn(V, K, generator=g) / 32
    dy = _softmax_grad(x, w, 40.0, 42)
    with pack.engine_scope(engine):
        gx, gw = _linear_grads(x, w, dy)
    dy64 = dy.double()
    ew, ex = _row_rel_l2(gw, dy64.t() @ x.double()), _row_rel_l2(gx, dy64 @ w.double())
    print(f"dW rows: worst rel L2 {ew.max().item():.3e}; dX rows: {ex.max().item():.3e}")
    assert ew.max().item() <= 1e-5 and ex.max().item() <= 1e-5


@gpu
@TIMEOUT
@pytest.mark.parametrize("engine", [pack.ENGINE_FFMA, pack.ENGINE_BF16X3, pack.ENGINE_F16X2, pack.ENGINE_F16],
                         ids=["ffma", "bf16x3", "f16x2", "f16"])
@pytest.mark.parametrize("M,K,V", [(256, 1024, 1024), (64, 256, 100)], ids=["tensor-core", "bmm"])
def test_training_gradients_scale_equivariant_bit_for_bit(engine, M, K, V):
    """Loss scaling must not change a gradient's bits: grads(dY * 2^k) == 2^k * grads(dY) for k = -40 and 20, on the
    tap-GEMM shape and on a shape that falls back to the fp32 batched matmul."""
    g = gen(M + K + V)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(V, K, generator=g) / 32
    dy = _softmax_grad(x, w, 10.0, 7)
    with pack.engine_scope(engine):
        base = _linear_grads(x, w, dy)
        for k in (-40, 20):
            f = 2.0 ** k
            got = _linear_grads(x, w, dy * f)
            for name, a, b in zip(("dX", "dW"), got, base):
                assert torch.equal(a, b * f), (name, k)


# ------------------------------------------------------------------------------------------ attention above the fp16 range
def _attn_ref(q, k, v, H):
    B, Tq, D = q.shape
    dh = D // H
    qh, kh, vh = (t.double().view(B, -1, H, dh).transpose(1, 2) for t in (q, k, v))
    s = qh @ kh.transpose(-1, -2) / math.sqrt(dh)
    return (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(B, Tq, D)


def _big_inputs(B, T, D, seed):
    g = gen(seed)
    q, k, v = (torch.randn(B, T, D, generator=g) for _ in range(3))
    return {"v*2^17": (q, k, v * 2.0 ** 17), "q*2^17,k*2^-17": (q * 2.0 ** 17, k * 2.0 ** -17, v)}


def _layer(D, H, seed):
    from megatts2_b200.modules.transformer import TransformerEncoderLayer
    lyr = TransformerEncoderLayer(dim=D, ff_dim=2 * D, conv_ff=False, n_heads=H)
    g = gen(seed)
    with torch.no_grad():
        for n, p in lyr.named_parameters():
            r = torch.randn(p.shape, generator=g)
            if "norm" in n:
                p.copy_(0.1 * r + (1.0 if n.endswith("weight") else 0.0))
            else:
                p.copy_(r / math.sqrt(p.shape[1]) if p.dim() == 2 else 0.1 * r)
    return lyr.to(DEV).eval()


def _layer_ref(lyr, x, H):
    P = {n: p.detach().cpu().double() for n, p in lyr.named_parameters()}
    D = x.shape[-1]
    x = x.double()
    ln = lambda t, i: F.layer_norm(t, (D,), P[f"norm{i}.weight"], P[f"norm{i}.bias"], 1e-5)
    lin = lambda t, n: t @ P[n + ".weight"].t() + P[n + ".bias"]
    h = ln(x, 1)
    a = _attn_ref(lin(h, "attn.w_q"), lin(h, "attn.w_k"), lin(h, "attn.w_v"), H)
    x = x + lin(a, "attn.out_proj.0")
    return x + lin(torch.relu(lin(ln(x, 2), "ff.0")), "ff.3")


def _scale_layer(lyr, which):
    with torch.no_grad():
        for n, f in ({"v*2^17": [("w_v", 2.0 ** 17)], "q*2^17,k*2^-17": [("w_q", 2.0 ** 17), ("w_k", 2.0 ** -17)]}[which]):
            getattr(lyr.attn, n).weight.mul_(f)
            getattr(lyr.attn, n).bias.mul_(f)
    pack.invalidate_plans()


def _maxerr(a, b):
    return (a.cpu().double() - b).abs().max().item()


def test_attention_entry_points_reject_null_params():
    """The full-range entry point and the fp16-range (tensor-core) one share the argument checks."""
    for fn in (L.lib().mtts_attention_f32, L.lib().mtts_attention_tc_f32):
        with pytest.raises(L.MttsError, match="null params"):
            L.check(fn(None, None))


@gpu
@TIMEOUT
@pytest.mark.parametrize("dh", [64, 96, 128])
@pytest.mark.parametrize("Tq", [70, 200])
def test_attention_above_fp16_range(Tq, dh):
    """bf16x3 and FFMA promise the fp32 range, so attention under them must be finite and fp32-grade for operands above
    65504 - through ops.attention and through the encoder driver.  Under the fp16-range engines (f16x2, f16) the range
    flag must be raised instead."""
    from megatts2_b200 import ops
    from megatts2_b200.modules.transformer import run_encoder
    dev = torch.device(DEV)
    B, H = 2, 4
    D = H * dh
    ops.tc_overflow_bind(dev)
    for name, (q, k, v) in _big_inputs(B, Tq, D, Tq + dh).items():
        ref = _attn_ref(q, k, v, H)
        for engine in (pack.ENGINE_BF16X3, pack.ENGINE_FFMA, pack.ENGINE_F16X2, pack.ENGINE_F16):
            ops.tc_overflow(dev)
            with pack.engine_scope(engine):
                y = ops.attention(q.to(DEV), k.to(DEV), v.to(DEV), H)
            if engine in (pack.ENGINE_BF16X3, pack.ENGINE_FFMA):
                assert bool(torch.isfinite(y).all()), (name, engine)
                assert _maxerr(y, ref) < 2e-5 * max(1.0, ref.abs().max().item()), (name, engine)
                assert not ops.tc_overflow(dev)
            else:
                assert ops.tc_overflow(dev), (name, engine)
        # the encoder driver (LN -> packed QKV GEMM -> attention -> out-projection -> FF), one layer of this width
        lyr = _layer(D, H, dh)
        x = torch.randn(B, Tq, D, generator=gen(5))
        _scale_layer(lyr, name)
        lref = _layer_ref(lyr, x, H)
        for engine in (pack.ENGINE_BF16X3, pack.ENGINE_FFMA, pack.ENGINE_F16X2, pack.ENGINE_F16):
            ops.tc_overflow(dev)
            with pack.engine_scope(engine):
                y = run_encoder(lyr, [lyr], x.to(DEV))
            if engine in (pack.ENGINE_BF16X3, pack.ENGINE_FFMA):
                assert bool(torch.isfinite(y).all()), (name, engine)
                err, scale = _maxerr(y, lref), max(1.0, lref.abs().max().item())
                assert err < 2e-5 * scale, (name, engine, err, scale)
            else:
                assert ops.tc_overflow(dev), (name, engine)


@gpu
@TIMEOUT
def test_synthesize_attention_overflow_reruns_finite_on_bf16x3(golden, weights_cpu):
    """An overflow that comes from attention (the first PLM layer's queries scaled by 2^17, its keys by 2^-17: the
    scores, and so the result, are unchanged in exact arithmetic): synthesize warns, reruns on bf16x3, and the rerun
    equals the unscaled model's bf16x3 result bit for bit."""
    from megatts2_b200 import ops
    dev = torch.device(DEV)
    g = golden("e2e")
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    phone = torch.randint(0, 320, (1, 70), generator=gen(13)).to(DEV)
    dur = torch.full((1, 70), 8, dtype=torch.int32, device=DEV)          # 560 frames: the PLM reaches 70 positions
    run = lambda: tts.synthesize(phone, g["mel_prompt"].to(DEV), forced_durations=dur, return_intermediates=True)
    with pack.engine_scope(pack.ENGINE_BF16X3):
        ref = run()
    _scale_layer(tts.plm.plm.layers[0], "q*2^17,k*2^-17")
    ops.tc_overflow(dev)
    with pack.engine_scope(pack.ENGINE_F16X2):
        with pytest.warns(UserWarning, match="fp16 range"):
            out = run()
    assert bool(torch.isfinite(out["wav"]).all())
    assert torch.equal(out["p_codes"], ref["p_codes"]) and torch.equal(out["wav"], ref["wav"])


# ------------------------------------------------------------------------------------------ plane writers, bit for bit
def _plan(fmt, M, K, N, ln, partial=64 << 20):
    out = (C.c_int32 * 5)()
    L.check(L.lib().mtts_tc_plan_query(132, 1, M, K, N, 1, 1, fmt, partial, ln, out))
    return dict(BN=out[0], splits=out[1])


def _params(x, w32, bias, y, B, Tin, Tout, Cin, Cout, k, dil=1, pad=0, pad_mode=0, pre_act=0):
    p = L.ConvParams()
    p.x, p.x_batch_stride, p.ldx = x.data_ptr(), Tin * Cin, Cin
    p.w, p.bias = w32.data_ptr(), bias.data_ptr() if bias is not None else None
    p.y = y.data_ptr() if y is not None else None
    p.B, p.Tin, p.Tout, p.Cin, p.Cout = B, Tin, Tout, Cin, Cout
    p.k, p.stride, p.dil, p.pad, p.pad_mode = k, 1, dil, pad, pad_mode
    p.pre_act, p.pre_slope, p.out_scale = pre_act, 0.1, 1.0
    return p


def _attach_tc(p, planes, rows, Cin, fmt):
    nbytes = 6 * rows * Cin + 4096
    scratch = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    p.w_tc, p.tc_scratch, p.tc_scratch_bytes, p.tc_fmt = planes.data_ptr(), scratch.data_ptr(), nbytes, fmt
    return scratch, planes          # the caller keeps both alive while the params point at them


def _run(p):
    from megatts2_b200 import ops
    ops.tc_overflow_bind(torch.device(DEV))
    L.check(L.lib().mtts_conv1d_f32(C.byref(p), ops._stream()))
    torch.cuda.synchronize()


def _fmt_ids(f):
    return FMT_NAMES[f]


@gpu
@TIMEOUT
@pytest.mark.parametrize("fmt", DEFAULT_FMTS, ids=_fmt_ids)
@pytest.mark.parametrize("pad_mode", [0, 1, 2], ids=["zero", "reflect", "replicate"])
def test_split_pad_planes_bit_exact(pad_mode, fmt):
    """The activation split of a convolution: the padded, pre-activated input as 3 - fmt planes equal to
    pack_tc_planes of it, halo rows included."""
    B, T, Cin, Cout, k, dil = 2, 300, 64, 64, 7, 3
    pad = dil * (k - 1) // 2
    g = gen(29 + pad_mode)
    x = torch.randn(B, T, Cin, generator=g) * 50
    w = torch.randn(Cout, Cin, k, generator=g) / 20
    y = torch.empty(B, T, Cout, device=DEV)
    xd = x.to(DEV)
    p = _params(xd, pack.pack_conv(w).to(DEV), None, y, B, T, T, Cin, Cout, k, dil, pad, pad_mode, L.ACT_LEAKY)
    p.y_batch_stride, p.ldy = T * Cout, Cout
    Tp = T + 2 * pad
    scratch, planes = _attach_tc(p, pack.pack_conv_tc_planes(w.to(DEV), fmt), B * Tp, Cin, fmt)
    _run(p)
    off = (-scratch.data_ptr()) % 1024
    n, npl = B * Tp * Cin, 3 - fmt
    got = scratch[off:off + 2 * n * npl].view(pack.plane_dtype(fmt)).view(npl, B * Tp, Cin)
    xt = F.leaky_relu(x, 0.1).transpose(1, 2)
    xt = F.pad(xt, (pad, pad), mode={1: "reflect", 2: "replicate"}[pad_mode]) if pad_mode else F.pad(xt, (pad, pad))
    assert torch.equal(_bits(got), _bits(pack.pack_tc_planes(xt.transpose(1, 2).reshape(B * Tp, Cin), fmt)))


@gpu
@TIMEOUT
@pytest.mark.parametrize("fmt", DEFAULT_FMTS, ids=_fmt_ids)
@pytest.mark.parametrize("Cin,Cout,k", [(256, 256, 3), (64, 64, 7), (32, 32, 11)], ids=["plain", "halo64", "halo32"])
def test_epilogue_next_layer_planes_bit_exact(Cin, Cout, k, fmt):
    """The tap-GEMM epilogue's plane output for the next layer: act(y) as 3 - fmt planes at the interior rows, equal to
    pack_tc_planes of the fp32 result the same epilogue stores; the halo rows stay untouched."""
    B, T, hl = 2, 700, 5
    g = gen(Cin + k + fmt)
    x = torch.randn(B, T, Cin, generator=g)
    w = torch.randn(Cout, Cin, k, generator=g) / math.sqrt(Cin)
    b = torch.randn(Cout, generator=g)
    pad = (k - 1) // 2
    y = torch.empty(B, T, Cout, device=DEV)
    xd = x.to(DEV)
    p = _params(xd, pack.pack_conv(w).to(DEV), b.to(DEV), y, B, T, T, Cin, Cout, k, 1, pad, 1, L.ACT_LEAKY)
    p.y_batch_stride, p.ldy = T * Cout, Cout
    keep = _attach_tc(p, pack.pack_conv_tc_planes(w.to(DEV), fmt), B * (T + 2 * pad), Cin, fmt)
    Tq, npl = T + 2 * hl, 3 - fmt
    out = torch.full((npl, B, Tq, Cout), 7.0, dtype=pack.plane_dtype(fmt), device=DEV)
    p.tc_out_planes, p.tc_out_plane_stride, p.tc_out_ld = out.data_ptr(), B * Tq * Cout, Cout
    p.tc_out_tp, p.tc_out_hl, p.tc_out_act, p.tc_out_slope = Tq, hl, L.ACT_LEAKY, 0.1
    _run(p)
    del keep
    spec = pack.pack_tc_planes(F.leaky_relu(y.cpu(), 0.1).reshape(B * T, Cout), fmt).view(npl, B, T, Cout)
    assert torch.equal(_bits(out[:, :, hl:hl + T]), _bits(spec))
    assert bool((out[:, :, :hl] == 7).all()) and bool((out[:, :, hl + T:] == 7).all())


@gpu
@TIMEOUT
@pytest.mark.parametrize("fmt", DEFAULT_FMTS, ids=_fmt_ids)
@pytest.mark.parametrize("dh", [64, 96, 128])
@pytest.mark.parametrize("Tq", [40, 130], ids=["fp32-kernel", "tc-kernel"])
def test_attention_plane_output_bit_exact(Tq, dh, fmt):
    """The attention's operand-plane output (the fused encoder feeds the out-projection with it) equals pack_tc_planes of
    the fp32 rows the same launch stores - from the fp32 kernel (Tq <= 64) and from the tensor-core kernel (Tq >= 65)."""
    from megatts2_b200 import ops
    B, H = 2, 2
    D = H * dh
    g = gen(Tq + dh + fmt)
    q, k, v = (torch.randn(B, Tq, D, generator=g).to(DEV) for _ in range(3))
    o = torch.empty(B, Tq, D, device=DEV)
    npl = 3 - fmt
    planes = torch.full((npl, B * Tq, D), 7.0, dtype=pack.plane_dtype(fmt), device=DEV)
    p = L.AttnParams()
    p.q, p.q_sb, p.q_st = q.data_ptr(), Tq * D, D
    p.k, p.k_sb, p.k_st = k.data_ptr(), Tq * D, D
    p.v, p.v_sb, p.v_st = v.data_ptr(), Tq * D, D
    p.o, p.o_sb, p.o_st = o.data_ptr(), Tq * D, D
    p.B, p.H, p.Tq, p.Tk, p.dh, p.scale = B, H, Tq, Tq, dh, 1.0 / math.sqrt(dh)
    p.o_planes, p.o_plane_stride, p.o_planes_ld, p.o_planes_fmt = planes.data_ptr(), B * Tq * D, D, fmt
    ops.tc_overflow_bind(torch.device(DEV))
    L.check(L.lib().mtts_attention_tc_f32(C.byref(p), ops._stream()))
    torch.cuda.synchronize()
    ref = _attn_ref(q.cpu(), k.cpu(), v.cpu(), H)
    assert _maxerr(o, ref) < 2e-5
    assert torch.equal(_bits(planes), _bits(pack.pack_tc_planes(o.cpu().reshape(B * Tq, D), fmt)))


def _check_scaled(y, ref, bar):
    err = (y.cpu().double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"err {err:.3e}  ({err / scale:.2e} of max|ref| = {scale:.3e})")
    assert err <= bar * scale, (err, scale)


@gpu
@TIMEOUT
@pytest.mark.parametrize("fmt", DEFAULT_FMTS, ids=_fmt_ids)
@pytest.mark.parametrize("M", [128, 192, 256])
def test_splitk_dense_default_formats(M, fmt):
    """Dense layers with too few output tiles split K across CTAs; the partial sums are reduced in a fixed order."""
    K, N = 4096, 1024
    g = gen(M + fmt)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g)
    ref = x.double() @ w.double().t() + b.double()
    xd = x.to(DEV)
    y = torch.empty(M, N, device=DEV)
    p = _params(xd, pack.pack_linear(w).to(DEV), b.to(DEV), y, 1, M, M, K, N, 1)
    p.ldy, p.y_batch_stride = N, 0
    keep = _attach_tc(p, pack.pack_tc_planes(w.to(DEV), fmt), M, K, fmt)
    part = torch.empty(8 * M * N, dtype=torch.float32, device=DEV)
    p.tc_partial, p.tc_partial_bytes = part.data_ptr(), part.numel() * 4
    assert _plan(fmt, M, K, N, 0, partial=part.numel() * 4)["splits"] > 1
    _run(p)
    _check_scaled(y, ref, 3e-5)
    y2 = torch.empty_like(y)
    p.y = y2.data_ptr()
    _run(p)
    del keep
    assert torch.equal(y, y2), "the split-K reduction order is fixed"


@gpu
@TIMEOUT
@pytest.mark.parametrize("fmt", DEFAULT_FMTS, ids=_fmt_ids)
@pytest.mark.parametrize("cin,cout,s,T,B", [(512, 256, 8, 100, 2), (128, 64, 2, 301, 3)])
def test_conv_transpose_default_formats(cin, cout, s, T, B, fmt):
    """The vocoder's up-samplers: ConvTranspose1d(k = 2s, stride s) as a 2-tap conv with s*Cout columns written at a
    negative out_shift, on the tensor cores."""
    g = gen(11 + s + fmt)
    x = torch.randn(B, T, cin, generator=g)
    w = torch.randn(cin, cout, 2 * s, generator=g) / math.sqrt(cin * 2)
    b = torch.randn(cout, generator=g)
    ref = F.conv_transpose1d(F.leaky_relu(x, 0.1).double().transpose(1, 2), w.double(), b.double(), stride=s,
                             padding=s // 2).transpose(1, 2)
    wp, bp = pack.pack_conv_transpose(w, b, s)
    xd, wp, bp = x.to(DEV), wp.to(DEV), bp.to(DEV)
    y = torch.empty(B, s * T, cout, device=DEV)
    p = _params(xd, wp, bp, y, B, T, T + 1, cin, s * cout, 2, pad=1, pre_act=L.ACT_LEAKY)
    p.y_batch_stride, p.ldy = s * T * cout, s * cout
    p.out_shift, p.y_batch_elems = -(s // 2) * cout, s * T * cout
    keep = _attach_tc(p, pack.pack_conv_transpose_tc_planes(wp, fmt), B * (T + 2), cin, fmt)
    _run(p)
    del keep
    _check_scaled(y, ref, 3e-5)


_LN_FUSE_SCRIPT = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}]
import helpers
from oracle import weights
plm = helpers.build_plm(weights.plm_state_dict(), "cuda")
x = torch.randn(8, 40, 1024, generator=torch.Generator().manual_seed(9)).cuda()
out = {{}}
for e in (1, 2):
    plm.plm.engine = e
    out[e] = plm.plm(x).cpu()
torch.save(out, {path!r})
"""


@gpu
@TIMEOUT
def test_splitk_layernorm_fusion_is_bit_identical_to_separate_launches(tmp_path):
    """At (B, T) = (8, 40) the encoder's dense layers split K and the reduction carries the next LayerNorm; that must
    equal the reduction + a separate LayerNorm launch (MEGATTS2_LN_FUSE=0, read once per process) bit for bit."""
    for fmt in DEFAULT_FMTS:
        assert _plan(fmt, 8 * 40, 4096, 1024, 1)["splits"] > 1
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    outs = []
    for i, fuse in enumerate(("1", "0")):
        path = str(tmp_path / f"enc{i}.pt")
        env = dict(os.environ, MEGATTS2_LN_FUSE=fuse)
        src = _LN_FUSE_SCRIPT.format(root=root, tests=os.path.join(root, "tests"), path=path)
        subprocess.run([sys.executable, "-c", src], check=True, env=env, cwd=root, timeout=300)
        outs.append(torch.load(path))
    for e in (1, 2):
        assert bool(torch.isfinite(outs[0][e]).all())
        assert torch.equal(outs[0][e], outs[1][e]), f"engine {e}"
