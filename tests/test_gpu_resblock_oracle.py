"""One dilation step of the fused ResBlock kernel (resblock_tc.cu, mtts_resblock_step_f32) against fp64, over the whole
shape domain the kernel accepts:

    y = (x + conv2(leaky(conv1_d(leaky(x)) + b1)) + b2) * out_scale (+ y_old)

The vocoder tests compare the kernel bit for bit with the two-launch tap-GEMM flow, which shares its reflection rule,
plane writer and epilogue arithmetic; here the reference is a plain restatement (F.pad reflect + F.conv1d in fp64), so a
mistake made the same way in both flows fails, and a kernel change that legitimately reorders its MMAs can be judged on
accuracy alone.

Bars, per element, built from convolutions of the products of each conv.  The per-product rounding errors are
independent, so they are summed as a root sum of squares (times LAMBDA, a Hoeffding tail) rather than in absolute value,
which would be sqrt(C k) times looser and could not tell a dropped correction term from rounding at k = 63:
  f16x2  fp64 over the exact operands: both operands split to 2^-22 (each product off by <= 2^-21 |w a|, plus the
         2^-36 floor), fp32 accumulation EPS_ACC * C k * sqrt(sum (w a)^2), conv1's bound carried through conv2 (leaky is
         1-Lipschitz), and the fp32 roundings of the epilogues.  The step without the f16x2 correction term is rejected
         in every case, and by 30x where C k is small enough for the accumulation allowance (checked on the host).
  f16    fp64 over the fp16-rounded operands (leaky(x).half(), w.half(), the intermediate .half()), as in
         test_gpu_f16_engine.py.  Only fp32 accumulation is left, plus one fp16 step of an intermediate that lies so
         close to a rounding midpoint that the kernel's fp32 value may round to the other neighbour.  That allowance is
         exact, so where such an intermediate did round the other way the error sits just below the bound.
The CPU tests at the top pin the eligibility rule and check that the case table reaches every buffer-ring configuration
and every per-CTA item-count class."""
import ctypes as C
import math
import os
import subprocess
import sys
import zlib

import pytest
import torch
import torch.nn.functional as F

import helpers
from megatts2_b200 import _lib as L
from megatts2_b200 import pack

DEV = "cuda"
gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16X2, F16 = L.TC_F16X2, L.TC_F16
FMT_NAME = {F16X2: "f16x2", F16: "f16"}
BAD_ARG, UNSUPPORTED = -1, -2

U = 2.0 ** -24                   # fp32 unit roundoff
EPS_ACC = U / 16                 # fp32 accumulation: EPS_ACC * (C k) * sqrt(sum (w a)^2)
SPLIT_EPS = 2.0 ** -21           # f16x2: each operand split to 2^-22 (leaky's fp32 rounding of x included)
SPLIT_FLOOR = 2.0 ** -15         # ... and below ~2^-36 lost (include/megatts2_b200.h)
LAMBDA = 6.0                     # independent rounding errors: P(|sum| > 6 sqrt(sum bound^2)) < 2 exp(-18) (Hoeffding)
SMS = (1, 2, 3, 0)               # SM budgets of ops.launch_policy; 0 = the whole device
FULL_SMS = 132                   # the H100 SXM's SM count, for the host-side item-count classes


def gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------ case table
def halos(k, dil):
    return dil * (k - 1) // 2, (k - 1) // 2


def rows_per_item(k):
    return 128 - (k - 1)                       # R = 128 - 2 h2 output rows per work item


def xbufs(C, fmt):
    """x-ring depth of the kernel's instantiation: two 48 KB buffers at C = 64 f16x2, else four"""
    return 2 if (C == 64 and fmt == F16X2) else 4


def _case(C, fmt, k, d, B, T, scale, acc):
    return dict(C=C, fmt=fmt, k=k, d=d, B=B, T=T, scale=scale, acc=acc)


def _cases():
    out = []
    ep = [(1.0, 0), (1 / 3, 1), (1.0, 1), (1 / 3, 0)]      # (out_scale, accumulate), cycled

    def add(C, fmt, k, d, B, T):
        s, a = ep[len(out) % len(ep)]
        out.append(_case(C, fmt, k, d, B, T, s, a))

    def R(k):
        return rows_per_item(k)

    # T classes (R = rows per item, h1 + h2 the two halos): shortest h1 + h2 + 1; T < R (one item reflected at both ends);
    # R, R + 1, 2R - 1, 2R, 2R + 1; R + h2 - 1 (the next-to-last item writes a tail reflection row); long (210 items)
    # ---- C = 32, f16x2 (x ring 4, staging 2)
    add(32, F16X2, 3, 1, 1, 128)                    # R + 2, B T = 128 exactly
    add(32, F16X2, 3, 1, 3, 50)                     # T < R
    add(32, F16X2, 3, 32, 3, R(3))                  # h1 = 32 edge, T = R
    add(32, F16X2, 17, 4, 3, R(17) + 8 - 1)         # h1 = 32 edge, R + h2 - 1
    add(32, F16X2, 17, 4, 1, 2 * R(17) - 1)
    add(32, F16X2, 63, 1, 3, 63)                    # k = 63 edge, shortest
    add(32, F16X2, 63, 1, 3, R(63) + 31 - 1)
    add(32, F16X2, 63, 1, 3, 70 * R(63))            # long
    add(32, F16X2, 7, 3, 1, 2 * R(7))
    add(32, F16X2, 5, 16, 1, 2 * R(5) + 1)          # h1 = 32 edge
    add(32, F16X2, 13, 2, 3, R(13) + 1)             # even h1 = 12, even h2 = 6
    # ---- C = 32, f16 (x ring 4, staging 2)
    add(32, F16, 11, 5, 3, R(11) + 5 - 1)
    add(32, F16, 11, 5, 3, 70 * R(11))              # long
    add(32, F16, 33, 2, 3, 49)                      # h1 = 32 edge, shortest
    add(32, F16, 33, 2, 1, 2 * R(33))
    add(32, F16, 3, 32, 3, R(3) + 1)                # h1 = 32 edge
    add(32, F16, 9, 8, 3, R(9))                     # h1 = 32 edge
    add(32, F16, 9, 8, 1, 2 * R(9) + 1)
    add(32, F16, 63, 1, 1, 2 * R(63) - 1)
    add(32, F16, 63, 1, 3, 63)
    add(32, F16, 15, 3, 3, 100)                     # odd h1 = 21, odd h2 = 7; T < R
    add(32, F16, 3, 3, 1, 2 * R(3) + 1)
    # ---- C = 64, f16x2 (x ring 2)
    add(64, F16X2, 3, 5, 1, 128)
    add(64, F16X2, 3, 31, 3, 60)                    # odd h1 = 31; T < R
    add(64, F16X2, 9, 8, 3, R(9) + 4 - 1)
    add(64, F16X2, 63, 1, 3, R(63) + 1)
    add(64, F16X2, 63, 1, 3, 70 * R(63))            # long
    add(64, F16X2, 17, 4, 1, 2 * R(17))
    add(64, F16X2, 33, 2, 1, 2 * R(33) + 1)
    add(64, F16X2, 33, 2, 3, 49)
    add(64, F16X2, 7, 1, 1, 2 * R(7) - 1)
    add(64, F16X2, 11, 3, 3, R(11))
    # ---- C = 64, f16 (x ring 4, staging 1)
    add(64, F16, 11, 1, 3, R(11))
    add(64, F16, 5, 16, 3, R(5) + 2 - 1)            # h1 = 32 edge
    add(64, F16, 5, 16, 3, 70 * R(5))               # long
    add(64, F16, 63, 1, 3, 63)
    add(64, F16, 63, 1, 1, 2 * R(63))
    add(64, F16, 31, 2, 3, 46)                      # even h1 = 30, odd h2 = 15; shortest
    add(64, F16, 31, 2, 1, 2 * R(31) + 1)
    add(64, F16, 3, 32, 3, R(3) + 1)
    add(64, F16, 17, 4, 1, 2 * R(17) - 1)
    add(64, F16, 7, 5, 3, 100)
    return out


CASES = _cases()


def case_id(c):
    sc = "s1" if c["scale"] == 1.0 else "s3"
    return f"C{c['C']}-{FMT_NAME[c['fmt']]}-k{c['k']}d{c['d']}-B{c['B']}T{c['T']}-{sc}a{c['acc']}"


def items_per_cta(c, sms):
    """per-CTA item counts: B ceil(T / R) items dealt round-robin over min(items, sms) CTAs"""
    items = c["B"] * -(-c["T"] // rows_per_item(c["k"]))
    ctas = min(items, sms)
    return {items // ctas, -(-items // ctas)}


# ------------------------------------------------------------------------------------------ fp64 reference
def _conv(a, w, dil):
    """'same' conv with reflect padding, (B, C, T) fp64"""
    h = dil * (w.shape[-1] - 1) // 2
    return F.conv1d(F.pad(a, (h, h), mode="reflect"), w, dilation=dil)


def inputs(c, seed=None):
    C_, k = c["C"], c["k"]
    g = gen(seed if seed is not None else zlib.crc32(case_id(c).encode()))
    x = torch.randn(c["B"], c["T"], C_, generator=g)
    w1 = torch.randn(C_, C_, k, generator=g) / math.sqrt(C_ * k)
    w2 = torch.randn(C_, C_, k, generator=g) / math.sqrt(C_ * k)
    b1 = torch.randn(C_, generator=g) * 0.1
    b2 = torch.randn(C_, generator=g) * 0.1
    y0 = torch.randn(c["B"], c["T"], C_, generator=g)
    return x, w1, b1, w2, b2, y0


def _rss(a, w, dil):
    """root sum of squares of the products of a 'same' conv: sqrt(sum_j,c (w a)^2), (B, C, T)"""
    return _conv(a * a, w * w, dil).sqrt()


def reference(x, w1, b1, w2, b2, dil, scale, acc, y0, fmt):
    """fp64 result of one step and its per-element error bound, both (B, T, C).  fmt F16: the computation over the
    fp16-rounded operands the f16 kernel multiplies; F16X2: over the exact operands."""
    s = float(torch.tensor(scale, dtype=torch.float32))           # the kernel multiplies by the fp32 value
    xt = x.double().transpose(1, 2)
    b1d, b2d = b1.double()[:, None], b2.double()[:, None]
    n = w1.shape[0] * w1.shape[-1]                                  # terms per output: C k
    acc_eps = EPS_ACC * n
    if fmt == F16:
        a = F.leaky_relu(x, 0.1).half().double().transpose(1, 2)  # leaky in fp32, then rounded, as the loader does
        w1d, w2d = w1.half().double(), w2.half().double()
    else:
        a = F.leaky_relu(xt, 0.1)
        w1d, w2d = w1.double(), w2.double()

    def conv_bound(a_, w_, d_):
        e = acc_eps * _rss(a_, w_, d_)
        if fmt == F16X2:      # each product off by <= 2^-21 |w a| + 2^-36 (|w| + |a|) <= 2^-21 (|w| + f)(|a| + f)
            e += LAMBDA * SPLIT_EPS * _rss(a_.abs() + SPLIT_FLOOR, w_.abs() + SPLIT_FLOOR, d_)
        return e

    c1 = _conv(a, w1d, dil) + b1d
    e1 = conv_bound(a, w1d, dil) + 4 * U * (c1.abs() + b1d.abs())
    m = F.leaky_relu(c1, 0.1)
    if fmt == F16:
        mh = m.half().double()
        # the kernel rounds its fp32 intermediate, within e1 of m: it may land one fp16 step away near a midpoint
        em = torch.maximum(((m - e1).half().double() - mh).abs(), ((m + e1).half().double() - mh).abs())
        m = mh
        carried = _conv(em, w2d.abs(), 1)                           # few and deterministic: summed in absolute value
    else:
        carried = LAMBDA * _rss(e1, w2d, 1)                         # leaky is 1-Lipschitz
    c2 = _conv(m, w2d, 1) + b2d
    e2 = conv_bound(m, w2d, 1) + carried + 4 * U * (c2.abs() + b2d.abs())
    v = c2 + xt
    out = v * s
    if acc:
        out = out + y0.double().transpose(1, 2)
    e = abs(s) * (e2 + U * (c2.abs() + v.abs())) + U * (v.abs() * abs(s) + out.abs())
    return out.transpose(1, 2), e.transpose(1, 2), m.transpose(1, 2)


# ------------------------------------------------------------------------------------------ CPU
ELIGIBLE = [
    # (B, T, C, k, dil, fmt) -> accepted
    ((1, 128, 32, 3, 1, F16X2), 1), ((1, 127, 32, 3, 1, F16X2), 0),        # B T = 128 is the least
    ((3, 43, 64, 3, 1, F16), 1), ((3, 42, 64, 3, 1, F16), 0),
    ((1, 2304, 64, 11, 5, F16X2), 1), ((2, 4608, 32, 7, 3, F16), 1),       # HiFi-GAN V1 stages
    ((1, 128, 64, 3, 32, F16X2), 1), ((1, 128, 64, 3, 33, F16X2), 0),      # h1 = d (k - 1) / 2 <= 32
    ((1, 128, 32, 5, 16, F16), 1), ((1, 128, 32, 5, 17, F16), 0),
    ((1, 128, 64, 9, 8, F16), 1), ((1, 128, 64, 9, 9, F16), 0),
    ((1, 128, 32, 17, 4, F16X2), 1), ((1, 128, 32, 17, 5, F16X2), 0),
    ((1, 128, 64, 33, 2, F16X2), 1), ((1, 128, 64, 33, 3, F16X2), 0),
    ((1, 128, 64, 63, 1, F16), 1), ((1, 200, 64, 65, 1, F16), 0),          # k <= 63
    ((1, 128, 32, 4, 1, F16X2), 0), ((1, 128, 32, 62, 1, F16X2), 0),       # odd k only
    ((1, 128, 32, 1, 1, F16X2), 0), ((1, 128, 32, 3, 0, F16X2), 0),        # k >= 3, dil >= 1
    ((3, 63, 64, 63, 1, F16X2), 1), ((3, 62, 64, 63, 1, F16X2), 0),        # T > h1 + h2
    ((3, 34, 32, 3, 32, F16), 0), ((3, 49, 32, 33, 2, F16), 1), ((3, 48, 32, 33, 2, F16), 0),
    ((1, 128, 16, 3, 1, F16X2), 0), ((1, 128, 128, 3, 1, F16X2), 0), ((1, 128, 48, 3, 1, F16), 0),   # C 32 | 64
    ((1, 128, 32, 3, 1, L.TC_BF16X3), 0), ((1, 128, 32, 3, 1, 3), 0),      # f16x2 | f16
]


def test_eligibility_boundary_table():
    lib = L.lib()
    for args, want in ELIGIBLE:
        assert lib.mtts_resblock_step_eligible(*args) == want, args


def test_case_table_reaches_every_ring_configuration_and_edge():
    lib = L.lib()
    for c in CASES:
        assert lib.mtts_resblock_step_eligible(c["B"], c["T"], c["C"], c["k"], c["d"], c["fmt"]) == 1, case_id(c)
    assert len({case_id(c) for c in CASES}) == len(CASES)
    # every (C, fmt) instantiation: odd and even per-CTA item counts, fewer than XBUFS (the ring never wraps) and more
    # than 2 XBUFS (every x-ring and weight-ring parity wraps)
    for C_ in (32, 64):
        for fmt in (F16X2, F16):
            xb = xbufs(C_, fmt)
            counts = set()
            for c in CASES:
                if (c["C"], c["fmt"]) == (C_, fmt):
                    for sms in SMS:
                        counts |= items_per_cta(c, sms or FULL_SMS)
            reach = dict(odd=any(n % 2 for n in counts), even=any(n % 2 == 0 for n in counts),
                         below_xbufs=any(n < xb for n in counts), above_2xbufs=any(n > 2 * xb for n in counts))
            assert all(reach.values()), (C_, FMT_NAME[fmt], reach)
    kd = {(c["k"], c["d"]) for c in CASES}
    v1 = {(k, d) for k in (3, 7, 11) for d in (1, 3, 5)}
    assert v1 <= kd
    assert {(3, 32), (5, 16), (9, 8), (17, 4), (33, 2), (63, 1)} <= kd                    # h1 = 32, k = 63
    assert {(halos(k, d)[0] % 2, halos(k, d)[1] % 2) for k, d in kd} == {(0, 0), (0, 1), (1, 1)}   # h2 even -> h1 even
    for C_ in (32, 64):
        for fmt in (F16X2, F16):
            assert any(c["k"] == 63 and (c["C"], c["fmt"]) == (C_, fmt) for c in CASES)
    classes = set()
    for c in CASES:
        T, R = c["T"], rows_per_item(c["k"])
        h1, h2 = halos(c["k"], c["d"])
        named = {"shortest": h1 + h2 + 1, "R": R, "R+1": R + 1, "2R-1": 2 * R - 1, "2R": 2 * R, "2R+1": 2 * R + 1}
        if h2 > 1:
            named["R+h2-1"] = R + h2 - 1
        classes |= {n for n, v in named.items() if v == T}
        if T < R:
            classes.add("T<R")
        if c["B"] * -(-T // R) >= 200:
            classes.add("long")
        if c["B"] * T == 128:
            classes.add("BT=128")
    assert classes == {"shortest", "T<R", "R", "R+1", "2R-1", "2R", "2R+1", "R+h2-1", "long", "BT=128"}, classes
    assert {c["B"] for c in CASES} == {1, 3}
    assert {(c["scale"], c["acc"]) for c in CASES} == {(1.0, 0), (1.0, 1), (1 / 3, 0), (1 / 3, 1)}


def test_f16x2_bar_sits_far_below_the_uncorrected_error():
    """Without its correction term an f16x2 step is the f16 step (one fp16 plane per operand): the f16x2 bar must reject
    that result in every case, and by 30x where the fp32 accumulation allowance (growing with C k) leaves room."""
    worst = {}
    for c in CASES:
        if c["fmt"] != F16X2 or c["B"] * c["T"] > 4000:
            continue
        x, w1, b1, w2, b2, y0 = inputs(c)
        ref, bound, _ = reference(x, w1, b1, w2, b2, c["d"], c["scale"], c["acc"], y0, F16X2)
        uncorrected, _, _ = reference(x, w1, b1, w2, b2, c["d"], c["scale"], c["acc"], y0, F16)
        worst[case_id(c)] = ((uncorrected - ref).abs() / bound).max().item()
    assert min(worst.values()) >= 4, worst
    assert max(worst.values()) >= 30, worst
    assert sum(r >= 30 for r in worst.values()) >= len(worst) // 3, worst


# ------------------------------------------------------------------------------------------ GPU: one step vs fp64
def _p(t):
    return C.c_void_p(t.data_ptr())


def step(x, y, w1p, b1, w2p, b2, c, stream=None):
    from megatts2_b200 import ops
    return L.lib().mtts_resblock_step_f32(_p(x), _p(y), _p(w1p), _p(b1), _p(w2p), _p(b2), c["B"], c["T"], c["C"], c["k"],
                                          c["d"], c["scale"], c["acc"], c["fmt"], stream or ops._stream())


def _device_args(x, w1, b1, w2, b2, fmt):
    return (x.to(DEV), pack.pack_conv_tc_planes(w1.to(DEV), fmt), b1.to(DEV), pack.pack_conv_tc_planes(w2.to(DEV), fmt),
            b2.to(DEV))


@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_resblock_step_vs_fp64(c):
    from megatts2_b200 import ops
    dev = torch.device(DEV)
    x, w1, b1, w2, b2, y0 = inputs(c)
    ref, bound, _ = reference(x, w1, b1, w2, b2, c["d"], c["scale"], c["acc"], y0, c["fmt"])
    xd, w1p, b1d, w2p, b2d = _device_args(x, w1, b1, w2, b2, c["fmt"])
    ops.tc_overflow(dev)                                            # binds and clears the range flag
    outs = []
    for sms in SMS:
        y = y0.to(DEV)                                              # accumulate 0 must overwrite it entirely
        with ops.launch_policy(sms):
            L.check(step(xd, y, w1p, b1d, w2p, b2d, c))
        torch.cuda.synchronize()
        outs.append(y.cpu())
    assert not ops.tc_overflow(dev), "the range flag was raised by in-range operands"
    for sms, o in zip(SMS[1:], outs[1:]):
        assert torch.equal(o, outs[0]), f"{sms} SMs differ from 1 SM: the result depends on the grid"
    err = (outs[0].double() - ref).abs()
    ratio = (err / bound).max().item()
    helpers.record(f"resblock_step_{FMT_NAME[c['fmt']]}", dict(case=case_id(c), err_to_bound=ratio,
                                                               max_err=err.max().item()))
    if ratio > 1:
        i = int((err / bound).argmax())
        b, t, ch = i // (c["T"] * c["C"]), (i // c["C"]) % c["T"], i % c["C"]
        pytest.fail(f"error {err.max().item():.3e} is {ratio:.2f}x the bound; worst at b={b} t={t} c={ch} "
                    f"(|err| {err[b, t, ch].item():.3e}, bound {bound[b, t, ch].item():.3e})")


# ------------------------------------------------------------------------------------------ GPU: fp16 range flag
def _intermediate_everywhere(x, w1, b1, dil, T_ext):
    """leaky(conv1 + b1) at positions [-h2, T_ext) the way the kernel computes its tile rows: x rows reflected once about
    the sequence ends (t < 0 -> -t, t >= T -> 2 (T - 1) - t), zeros where that is still outside."""
    B, T, C_ = x.shape
    k = w1.shape[-1]
    h1, h2 = halos(k, dil)
    pos = torch.arange(-h1 - h2, T_ext + h1)
    src = torch.where(pos < 0, -pos, pos)
    src = torch.where(src >= T, 2 * (T - 1) - src, src)
    inside = (src >= 0) & (src < T)
    a = F.leaky_relu(x.double(), 0.1)[:, src.clamp(0, T - 1)] * inside[None, :, None]
    c1 = F.conv1d(a.transpose(1, 2), w1.double(), b1.double(), dilation=dil)
    return F.leaky_relu(c1, 0.1).transpose(1, 2)                   # position p at index p + h2


@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("C_,fmt", [(32, F16X2), (32, F16), (64, F16X2), (64, F16)])
def test_range_flag_is_raised_exactly_for_interior_rows(C_, fmt):
    """The flag is raised exactly when an interior row (t in [0, T)) of leaky(x), or of leaky(conv1 + b1), is beyond 65504.
    Rows the kernel computes past the sequence end (replaced by reflections, or discarded) never raise it."""
    from megatts2_b200 import ops
    dev = torch.device(DEV)
    k, d = 7, 3
    h1, h2 = halos(k, d)
    R = rows_per_item(k)
    T = R + 10                                                      # the last item holds 10 rows
    c = _case(C_, fmt, k, d, 1, T, 1.0, 0)
    g = gen(C_ + fmt)
    x0 = torch.randn(1, T, C_, generator=g)
    w0 = torch.randn(C_, C_, k, generator=g) / math.sqrt(C_ * k)
    b1 = torch.zeros(C_)                                            # leaky(a z) = a leaky(z): the intermediate scales with w1
    w2, b2 = w0.flip(0), torch.zeros(C_)
    LIM = 65504.0

    def flag(x, w1):
        xd, w1p, b1d, w2p, b2d = _device_args(x, w1, b1, w2, b2, fmt)
        y = torch.empty_like(xd)
        ops.tc_overflow(dev)
        L.check(step(xd, y, w1p, b1d, w2p, b2d, c))
        return ops.tc_overflow(dev)

    def interior_max(x, w1):
        m = _intermediate_everywhere(x, w1, b1, d, T + 128)
        return m[:, h2:h2 + T].abs().max().item(), m

    m0, _ = interior_max(x0, w0)
    assert not flag(x0, w0)
    # the intermediate: clearly above and clearly below the limit at its largest interior element
    assert flag(x0, w0 * (1.5 * LIM / m0))
    assert not flag(x0, w0 * (0.5 * LIM / m0))
    # leaky(x): one interior element above / below the limit (negative x is scaled by 0.1), the intermediate kept small
    p = T // 2
    for v, want in ((7.0e4, True), (6.0e4, False), (-7.0e4, False), (-7.0e5, True)):
        x = x0.clone()
        x[0, p, 3] = v
        w1 = w0 * 1e-3
        assert interior_max(x, w1)[0] < 0.5 * LIM
        assert flag(x, w1) == want, v
    # an intermediate row past the end that the last item computes (position q = p + h1 >= T, which reads x[p] through
    # tap 0 only) far beyond the limit, every interior row far below it: the flag stays clear
    p = T - 3
    q = p + h1
    x = x0 * 0.01
    x[0, p] = 1000.0
    w1 = w0 * 0.1
    w1[:, :, 0] = torch.randn(C_, C_, generator=g) * (3.0e5 / (1000.0 * math.sqrt(C_)))
    top, m = interior_max(x, w1)
    assert top < 0.5 * LIM and m[0, q + h2].abs().max().item() > 2 * LIM, (top, m[0, q + h2].abs().max().item())
    assert q < (T // R) * R - h2 + 128                              # inside the last item's tile
    assert not flag(x, w1)


# ------------------------------------------------------------------------------------------ GPU: refusals
@gpu
@pytest.mark.timeout(300)
def test_refusals_launch_nothing():
    from megatts2_b200 import ops
    dev = torch.device(DEV)
    ops.tc_overflow_bind(dev)
    n_elem = 3 * 256 * 128
    buf_x = torch.randn(n_elem + 16, device=DEV)
    buf_y = torch.zeros(n_elem + 16, device=DEV)
    w = torch.zeros(2 * 65 * 128 * 128, dtype=torch.float16, device=DEV)
    b = torch.zeros(128 + 16, device=DEV)
    refused = [
        _case(32, F16X2, 3, 33, 1, 200, 1.0, 0),      # h1 = 33
        _case(64, F16, 65, 1, 1, 200, 1.0, 0),        # k = 65
        _case(32, F16X2, 4, 1, 1, 200, 1.0, 0),       # even k
        _case(64, F16X2, 63, 1, 3, 62, 1.0, 0),       # T = h1 + h2
        _case(32, F16, 3, 1, 1, 127, 1.0, 0),         # B T = 127
        _case(16, F16X2, 3, 1, 1, 200, 1.0, 0),
        _case(128, F16, 3, 1, 1, 200, 1.0, 0),
        dict(_case(32, F16X2, 3, 1, 1, 200, 1.0, 0), fmt=L.TC_BF16X3),
    ]
    n0 = ops.launch_count()
    for c in refused:
        assert step(buf_x, buf_y, w, b, w, b, c) == UNSUPPORTED, c
    ok = _case(32, F16X2, 3, 1, 1, 200, 1.0, 0)
    assert step(buf_x, buf_x, w, b, w, b, ok) == BAD_ARG                                  # x == y
    x4, y4, b4 = buf_x[1:], buf_y[1:], b[1:]                                              # 4-byte offsets
    assert step(x4, buf_y, w, b, w, b, ok) == BAD_ARG
    assert step(buf_x, y4, w, b, w, b, ok) == BAD_ARG
    assert step(buf_x, buf_y, w, b4, w, b, ok) == BAD_ARG
    assert step(buf_x, buf_y, w, b, w, b4, ok) == BAD_ARG
    torch.cuda.synchronize()
    assert ops.launch_count() == n0, "a refused call launched a kernel"
    assert bool((buf_y == 0).all())


# ------------------------------------------------------------------------------------------ GPU: the vocoder around it
# two stages: C = 64 at L = 2 (T + 10), C = 32 at L = 4 (T + 10)
_SMALL = dict(upsample_initial_channel=128, upsample_factors=(2, 2), upsample_kernel_sizes=(4, 4))
VOCODERS = {
    # ResBlocks at the h1 = 32 and k = 63 edges, with even and odd halos
    "edges_a": dict(_SMALL, resblock_kernel_sizes=(5, 9, 63), resblock_dilation_sizes=((1, 16, 2), (1, 8, 3), (1, 1, 1))),
    "edges_b": dict(_SMALL, resblock_kernel_sizes=(3, 17, 33), resblock_dilation_sizes=((1, 32, 5), (1, 4, 2), (2, 2, 1))),
    # h1 = 33 is not eligible: both stages keep the two-launch flow
    "fallback_d33": dict(_SMALL, resblock_kernel_sizes=(3, 7), resblock_dilation_sizes=((1, 33, 2), (1, 3, 5))),
}
VOC_B, VOC_T = 2, 40
VOC_BAR = 2e-6                  # fp32-grade through the whole vocoder: 2e-7 observed on an H100 (f16x2 and bf16x3)


def build_vocoder(name):
    """HifiganGenerator with seeded weights, scaled so that the fp64 signal before tanh stays inside +-1"""
    from megatts2_b200.models.megatts2 import HifiganGenerator
    gen_ = HifiganGenerator(**VOCODERS[name])
    g = gen(7)
    with torch.no_grad():
        for p in gen_.parameters():
            if p.dim() > 1:
                p.copy_(torch.randn(p.shape, generator=g) * (0.5 / p[0].numel() ** 0.5))
            else:
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
        gen_.conv_post.weight.mul_(0.5)
    mel = torch.randn(VOC_B, 80, VOC_T, generator=gen(11)) * 2 - 4
    return gen_, mel


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", list(VOCODERS))
def test_vocoder_edges_vs_fp64_oracle(name):
    from megatts2_b200.models.megatts2 import HIFIGAN
    from oracle import ref_megatts2 as R
    gen_, mel = build_vocoder(name)
    sd64 = {k: v.detach().double() for k, v in gen_.state_dict().items()}
    ref = R.hifigan_generator(sd64, mel.double(), gen_.cfg)
    assert ref.abs().max().item() < math.tanh(1.0), "the signal before tanh leaves +-1: scale the weights down"
    h = HIFIGAN(gen_.to(DEV)).eval()
    for engine in (pack.ENGINE_F16X2, pack.ENGINE_BF16X3):
        h.generator.engine = engine
        wav = h.decode_batch(mel.to(DEV))
        torch.cuda.synchronize()
        err = (wav.cpu().double() - ref).abs().max().item()
        helpers.record("resblock_vocoder", dict(config=name, engine=engine, max_err=err))
        assert err < VOC_BAR, (name, engine, err)


_SCRIPT = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}]
import test_gpu_resblock_oracle as t
from megatts2_b200 import ops, pack
from megatts2_b200.models.megatts2 import HIFIGAN
dev = torch.device("cuda", 0)
out = {{}}
for name in t.VOCODERS:
    gen_, mel = t.build_vocoder(name)
    h = HIFIGAN(gen_.to(dev)).eval()
    h.generator.engine = pack.ENGINE_F16X2
    ops.tc_overflow(dev)
    n0 = ops.launch_count()
    wav = h.decode_batch(mel.to(dev))
    torch.cuda.synchronize()
    out[name] = (wav.cpu(), ops.tc_overflow(dev), ops.launch_count() - n0)
torch.save(out, {path!r})
"""


def _run(fuse, tmp_path):
    path = str(tmp_path / f"rbo{fuse}.pt")
    src = _SCRIPT.format(root=ROOT, tests=os.path.join(ROOT, "tests"), path=path)
    subprocess.run([sys.executable, "-c", src], check=True, env=dict(os.environ, MEGATTS2_RB_FUSE=fuse), cwd=ROOT,
                   timeout=600)
    return torch.load(path)


@gpu
@pytest.mark.timeout(900)
def test_vocoder_edges_fused_is_bit_identical_to_two_launch_flow(tmp_path):
    fused, plain = _run("1", tmp_path), _run("0", tmp_path)
    for name in VOCODERS:
        (wf, of, nf), (wp, op, np_) = fused[name], plain[name]
        if name.startswith("fallback"):
            assert nf == np_, f"{name}: an ineligible dilation step must keep the stage on two launches ({nf} vs {np_})"
        else:
            assert nf < np_, f"{name}: the fused path did not run ({nf} vs {np_} launches)"
        assert not of and not op, name
        assert torch.equal(wf, wp), f"{name}: max diff {(wf - wp).abs().max().item()}"
