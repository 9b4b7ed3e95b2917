"""Both inference attention kernels against fp64, at every instantiation attention() (csrc/ops.cu) can launch:

    o = softmax(q k^T * scale + mask) v          per (batch item, head, query row)

  fp32   attn_kernel<NI, RW, NW, KPL> (ops.cu): FMA dot products in d order, online softmax over 32 KPL-key tiles, the
         P V product as an FMA chain in key order.  dh 64 / 96 / 128 with RW = ceil(Tq / 8) <= 8 and KPL = 2 when Tk > 32
         (48 instantiations), <8, 4, 4, 1> (dh 256) and <16, 4, 4, 1> (dh 512); each with a 16-byte and a scalar load path.
  tc     attn_tc_kernel<64 | 96 | 128> (attn_tc.cu): Q, K, V and P split into f16x2 planes, three wgmmas per product, 64-key
         tiles.  Reached by the fp16-range entry point for Tq >= 65, and for AR steps (Tq == Tk <= 64, even H, dh 64 / 96)
         once mtts_set_attention_pair_min allows it.
Which one a case runs on is read from mtts_attention_plan_query, the routing rule attention() itself dispatches from.

The reference is fp64 over the exact fp32 inputs (the fp32 value of scale included).  Bars, per output element, come from
a first-order perturbation of the softmax.  With the reference's p_j and o of a row, an error d_j in score j moves the
output by sum_j p_j d_j (v_jd - o_d), an error of p_j's exponential by the same with d_j its relative error, so

    |do_d| <= sum_j p_j (E_s,j + E_exp,j) |v_jd - o_d|  +  E_pv,d  +  E_norm,d

  E_s,j   the score error.  fp32: the dh-term FMA chain rounds each running sum S_i once, so the error is at most
          u sum_i |S_i|; the roundings are independent, so also LAMBDA u sqrt(sum_i S_i^2) (the smaller is used), times
          scale.  Then one rounding each for the product with scale, the mask add and the subtraction of the row max:
          u (|x| + |x + mask| + |x + mask - m|).  tc: each product q_d k_d is off by <= SPLIT_EPS (|q_d| + f)(|k_d| + f)
          (both operands split to 2^-22, the 2^-36 floor; f = SPLIT_FLOOR), summed as above (absolute, or LAMBDA times
          the root sum of squares), plus the accumulation: ASSUMED (wgmma's accumulation rounding is not documented) to
          lose at most 2u of the running sum and of the 16 products of each k-step, 2u (sum_ks |S_ks| + sum_d |q_d k_d|).
          The main + correction recombination adds one more u |x|.
  E_exp   expf is within 2 ulp (4u) for each p_j; each later online-softmax rescale alpha = expf(m_old - m_new) adds 4u
          and u |m_new - m_old| for the keys of the tiles before it (a rescale from -inf is exactly 0).
  E_pv    the P V accumulation.  fp32: an FMA chain in key order, each running sum O_j rounded once (min of u sum_j |O_j|
          and LAMBDA u sqrt(sum_j O_j^2)), plus one rounding of the accumulator per rescale.  tc: V and P split like the
          score operands (P unnormalised in [0, 1], so p below ~2^-36 vanishes: the floor term), the ASSUMED 2u per
          16-key k-step as above, and the rescales.
  E_norm  l sums positive terms (each lane's keys, a 5-level warp butterfly or a 2-level quad shuffle, two roundings per
          tile), so its relative error is at most its addition depth times u; 1 / l and the products add 3 (tc 4) more,
          all times |o_d|.
u = U = 2^-24.  SPLIT_EPS, SPLIT_FLOOR and LAMBDA are those of test_gpu_resblock_oracle.py.  The CPU test
test_bar_rejects_plausible_wrong_kernels checks that the bars have teeth: the tc kernel without its f16x2 correction terms
(Q, K, V and P each rounded once to fp16) and the fp32 kernel on TF32-rounded operands both exceed every case's bar by
at least 4x.

The CPU tests at the top pin the routing rule at its edges and check that the case table reaches every instantiation and
the scalar load path of every head dim.  The GPU tests also check, per case, what must hold bit for bit: a repeat launch,
one item of a batched launch against a single-item launch, and the operand-plane output (bf16x3, f16x2) against
pack_tc_planes of the fp32 rows of the same launch."""
import ctypes as C
import functools
import math
import zlib

import pytest
import torch

import helpers
from megatts2_b200 import _lib as L
from megatts2_b200 import pack
from test_gpu_resblock_oracle import LAMBDA, SPLIT_EPS, SPLIT_FLOOR, U

DEV = "cuda"
gpu = pytest.mark.gpu
BAD_ARG, UNSUPPORTED = -1, -2
NONE, FP32, TC, PAIR = -1, 0, 1, 2                     # MTTS_ATTN_*
KNAME = {NONE: "none", FP32: "fp32", TC: "tc", PAIR: "tc-pair"}
OFF = 0                                                 # pair_min: AR-step routing off


def gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------ case table
def _case(dh, H, B, Tq, Tk, entry="f32", mask="none", layout="contig", mag="randn", pair=OFF):
    return dict(dh=dh, H=H, B=B, Tq=Tq, Tk=Tk, entry=entry, mask=mask, layout=layout, mag=mag, pair=pair)


def _cases():
    out = []
    mags = ("randn", "peaky", "flat")

    def add(dh, H, B, Tq, Tk, **kw):
        kw.setdefault("mag", mags[len(out) % 3])
        if kw.get("mask", "").startswith("pad") or kw.get("mask") == "causalpad":
            B = max(B, 3)                               # lengths: full, ending inside a key tile, ending at a tile edge
        out.append(_case(dh, H, B, Tq, Tk, **kw))

    # ---- fp32 kernel, dh 64 / 96 / 128: one Tq per RW class, each with Tk = Tq and a Tk on the other side of 32
    H_OF = {64: 16, 96: 8, 128: 4}
    sq_masks = ("causal", "edge", "pad", "rand", "none", "edge1e9", "pad1e9")
    sq_lay = ("packed", "contig", "strided_o", "misaligned")
    x_masks = ("edge", "pad", "rand", "edge1e9", "none", "pad1e9")
    x_lay = ("contig", "strided_o", "misaligned")
    lo, hi = (1, 31, 32), (65, 300, 33, 63, 64)
    n = 0
    for dh in (64, 96, 128):
        for Tq in (1, 9, 17, 25, 33, 41, 49, 57, 64):
            add(dh, H_OF[dh], 2, Tq, Tq, entry=("f32", "tc")[n % 2], mask=sq_masks[n % 7], layout=sq_lay[n % 4])
            Tk = hi[n % 5] if Tq <= 32 else lo[n % 3]
            add(dh, H_OF[dh], 2, Tq, Tk, entry=("tc", "f32")[n % 2], mask=x_masks[n % 6], layout=x_lay[n % 3])
            n += 1
    # ---- fp32 kernel through the full-range entry point at Tq >= 65: several query CTAs
    for dh in (64, 96, 128):
        for t, Tk in enumerate((1, 31, 32, 33, 63, 64, 65, 300)):
            add(dh, 2, 2, (65, 130, 200)[(t + dh) % 3], Tk, mask=x_masks[t % 6], layout=x_lay[(t + dh) % 3])
        T = {64: 65, 96: 130, 128: 200}[dh]
        add(dh, 2, 2, T, T, mask="causal", layout="packed")
    # ---- fp32 kernel, dh 256 (MRTE phone encoder, 2 heads) and dh 512 (MRTE cross-attention, 1 head)
    for dh, H in ((256, 2), (512, 1)):
        for a, Tq in enumerate((1, 16, 17, 70)):
            for b, Tk in enumerate((1, 32, 33, 100, 257)):
                i = 5 * a + b
                add(dh, H, 2, Tq, Tk, entry=("f32", "tc")[i % 2], mask=x_masks[(i + dh // 256) % 6],
                    layout=x_lay[i % 3])
        add(dh, H, 2, 33, 33, entry="tc", mask="causal", layout="packed")
        add(dh, H, 2, 70, 70, mask="edge", layout="misaligned")
    # ---- tc kernel (Tq >= 65), square and cross shapes; a misaligned base falls back to the fp32 kernel's scalar path
    tc_shapes = ((65, 65, "causal", "packed"), (128, 1, "rand", "contig"), (129, 7, "pad", "strided_o"),
                 (200, 64, "edge1e9", "contig"), (65, 300, "edge", "strided_o"), (128, 128, "pad1e9", "packed"),
                 (129, 65, "edge", "contig"), (200, 200, "causal", "strided_o"), (200, 300, "rand", "misaligned"),
                 (65, 100, "none", "contig"))
    for dh in (64, 96, 128):
        for Tq, Tk, m, lay in tc_shapes:
            add(dh, 8 if Tq * Tk <= 65 * 65 else 4 if Tq * Tk < 200 * 200 else 2, 2, Tq, Tk, entry="tc", mask=m,
                layout=lay)
    # ---- tc kernel through the AR-step route (Tq == Tk <= 64, even H)
    for dh, H in ((64, 16), (96, 8)):
        for T, m, lay in ((16, "causal", "packed"), (33, "edge", "contig"), (64, "pad", "strided_o"),
                          (33, "causal", "packed"), (64, "rand", "contig")):
            add(dh, H, 2, T, T, entry="tc", mask=m, layout=lay, pair=16)
    # ---- the KV-cache decode step (Tq = 1, K / V rows of a cache with room for more) and the last-row layer
    for dh, H, Tk, entry in ((64, 16, 1, "f32"), (64, 16, 32, "tc"), (64, 16, 33, "f32"), (64, 16, 300, "tc"),
                             (96, 8, 17, "tc"), (96, 8, 64, "f32"), (96, 8, 65, "tc")):
        add(dh, H, 2, 1, Tk, entry=entry, layout="decode")
    for dh, H, T, m, entry in ((64, 16, 40, "causalpad", "f32"), (96, 8, 70, "pad", "tc"), (64, 16, 300, "causalpad", "tc"),
                               (96, 8, 33, "causalpad", "f32")):
        add(dh, H, 2, 1, T, entry=entry, mask=m, layout="lastrow")
    return out


CASES = _cases()


def case_id(c):
    pair = f"-pair{c['pair']}" if c["pair"] else ""
    return (f"dh{c['dh']}-H{c['H']}B{c['B']}-q{c['Tq']}k{c['Tk']}-{c['entry']}{pair}-{c['mask']}-{c['layout']}-"
            f"{c['mag']}")


def intended_plan(c):
    """the routing rule, restated: (kernel, dh, RW, NW, KPL, vec)"""
    dh, Tq, Tk = c["dh"], c["Tq"], c["Tk"]
    vec = int(c["layout"] != "misaligned")
    if c["entry"] == "tc" and vec and dh in (64, 96, 128):
        if Tq >= 65:
            return (TC, dh, 0, 0, 0, 1)
        if c["pair"] and Tq >= c["pair"] and Tq == Tk <= 64 and c["H"] % 2 == 0 and dh in (64, 96):
            return (PAIR, dh, 0, 0, 0, 1)
    if dh in (256, 512):
        return (FP32, dh, 4, 4, 1, vec)
    return (FP32, dh, 8 if Tq >= 64 else -(-Tq // 8), 8, 2 if Tk > 32 else 1, vec)


def key_tile(plan):
    return 32 * plan[4] if plan[0] == FP32 else 64


def plan_str(plan):
    k, dh, rw, nw, kpl, vec = plan
    if k == FP32:
        return f"attn_kernel<{dh // 32},{rw},{nw},{kpl}>{'' if vec else ' scalar'}"
    return f"attn_tc_kernel<{dh}>{' (pair route)' if k == PAIR else ''}"


# ------------------------------------------------------------------------------------------ layouts and masks
def _layout(c):
    """buffers (name -> floats) and the views of q, k, v, o: (buffer, offset, batch stride, row stride), in floats"""
    B, Tq, Tk, D = c["B"], c["Tq"], c["Tk"], c["H"] * c["dh"]
    lay = c["layout"]
    if lay == "packed":
        assert Tq == Tk
        bufs = dict(qkv=B * Tq * 3 * D)
        views = dict(q=("qkv", 0, 3 * D * Tq, 3 * D), k=("qkv", D, 3 * D * Tq, 3 * D), v=("qkv", 2 * D, 3 * D * Tq, 3 * D))
    elif lay == "decode":                               # q: this step's qkv row; k / v: a cache of Tk + 7 rows of [k | v]
        assert Tq == 1
        Ta = Tk + 7
        bufs = dict(qkv=B * 3 * D, kv=B * Ta * 2 * D)
        views = dict(q=("qkv", 0, 3 * D, 3 * D), k=("kv", 0, Ta * 2 * D, 2 * D), v=("kv", D, Ta * 2 * D, 2 * D))
    elif lay == "lastrow":                              # q: row T - 1 of the layer's packed qkv
        assert Tq == 1
        T = Tk
        bufs = dict(qkv=B * T * 3 * D)
        views = dict(q=("qkv", (T - 1) * 3 * D, 3 * D * T, 3 * D), k=("qkv", D, 3 * D * T, 3 * D),
                     v=("qkv", 2 * D, 3 * D * T, 3 * D))
    else:
        m = int(lay == "misaligned")                    # a 4-byte offset base pointer
        bufs = dict(q=B * Tq * D + m, k=B * Tk * D + m, v=B * Tk * D + m)
        views = dict(q=("q", m, Tq * D, D), k=("k", m, Tk * D, D), v=("v", m, Tk * D, D))
    if lay == "strided_o":
        bufs["o"] = B * Tq * (D + 32)
        views["o"] = ("o", 0, Tq * (D + 32), D + 32)
    else:
        bufs["o"] = B * Tq * D
        views["o"] = ("o", 0, Tq * D, D)
    return bufs, views


def pad_lengths(Tk, tile, B):
    inside = min(Tk, tile + tile // 2 + 1) if Tk > tile else max(1, (Tk + 1) // 2)
    edge = tile * ((Tk - 1) // tile) if Tk > tile else inside
    return [(Tk, inside, edge)[b % 3] for b in range(B)]


def make_mask(c, tile, g):
    """the stored additive mask, its element strides (sb, sh, sq) and the offset the kernel is given, or None"""
    kind, B, H, Tq, Tk = c["mask"], c["B"], c["H"], c["Tq"], c["Tk"]
    if kind == "none":
        return None
    neg = -1e9 if kind.endswith("1e9") else float("-inf")
    if kind == "causal":
        assert Tq == Tk
        m = torch.full((Tq, Tk), float("-inf")).triu(1).expand(B, H, Tq, Tk).contiguous()
        return m, (H * Tq * Tk, Tq * Tk, Tk), 0
    if kind.startswith("pad"):                          # (B, 1, 1, Tk) broadcast over heads and rows
        m = torch.zeros(B, 1, 1, Tk)
        for b, n in enumerate(pad_lengths(Tk, tile, B)):
            m[b, ..., n:] = neg
        return m, (Tk, 0, 0), 0
    if kind == "causalpad":                             # (B, 1, T, T), last row only: the pointer moves by (T - 1) mask_sq
        T = Tk
        m = torch.full((T, T), float("-inf")).triu(1).expand(B, 1, T, T).contiguous()
        for b, n in enumerate(pad_lengths(T, tile, B)):
            m[b, ..., n:] = float("-inf")
        return m, (T * T, 0, T), (T - 1) * T
    if kind == "rand":
        return torch.randn(B, H, Tq, Tk, generator=g) * 2, (H * Tq * Tk, Tq * Tk, Tk), 0
    assert kind.startswith("edge")
    m = torch.randn(B, H, Tq, Tk, generator=g) * 0.5
    for i in range(Tq):
        if i % 3 == 0 and Tk > tile:
            m[:, :, i, :tile] = neg                     # the row's whole first key tile
        elif i % 3 == 1 and Tk > 1:
            m[:, :, i, :-1] = neg                       # everything but the row's last key
    return m, (H * Tq * Tk, Tq * Tk, Tk), 0


def logical_mask(stored, B, H, Tq, Tk):
    if stored is None:
        return None
    m, (sb, sh, sq), off = stored
    return torch.as_strided(m.reshape(-1), (B, H, Tq, Tk), (sb, sh, sq, 1), off)


@functools.lru_cache(maxsize=None)
def inputs(cid):
    """q (B, Tq, D), k / v (B, Tk, D), the stored mask and its logical (B, H, Tq, Tk) view; the mask is laid out for the
    kernel the case was written for"""
    c = CASE_BY_ID[cid]
    g = gen(zlib.crc32(cid.encode()))
    B, Tq, Tk, D = c["B"], c["Tq"], c["Tk"], c["H"] * c["dh"]
    qs = {"randn": 1.0, "peaky": 20.0, "flat": 1e-3}[c["mag"]]
    q = torch.randn(B, Tq, D, generator=g) * qs
    k = torch.randn(B, Tk, D, generator=g)
    v = torch.randn(B, Tk, D, generator=g)
    stored = make_mask(c, key_tile(intended_plan(c)), g)
    return q, k, v, stored, logical_mask(stored, B, c["H"], Tq, Tk)


CASE_BY_ID = {case_id(c): c for c in CASES}


# ------------------------------------------------------------------------------------------ fp64 reference and bar
def _heads(t, H):
    B, T, D = t.shape
    return t.double().view(B, T, H, D // H).transpose(1, 2)


def _split_sum(a, b, dim):
    """sum of the split-error bounds SPLIT_EPS (|a| + f)(|b| + f) over `dim`: the smaller of the absolute sum and LAMBDA
    times the root sum of squares"""
    t = (a.abs() + SPLIT_FLOOR) * (b.abs() + SPLIT_FLOOR)
    return SPLIT_EPS * torch.minimum(t.sum(dim), LAMBDA * t.square().sum(dim).sqrt())


def _fma_chain(S, dim):
    """an FMA chain whose running sums are S: the smaller of u sum |S| and LAMBDA u sqrt(sum S^2)"""
    return U * torch.minimum(S.abs().sum(dim), LAMBDA * S.square().sum(dim).sqrt())


def _head_ref(Q, K, V, M, scale, plan):
    """one (batch item, head): Q (Tq, dh), K / V (Tk, dh), M (Tq, Tk) or None -> o and its bar, (Tq, dh)"""
    kernel, kpl = plan[0], plan[4]
    Tq, dh = Q.shape
    Tk = K.shape[0]
    tile = key_tile(plan)
    nkt = -(-Tk // tile)
    dot = Q @ K.T
    x = dot * scale
    xm = x + M if M is not None else x
    m = xm.max(-1, keepdim=True).values
    e = torch.exp(xm - m)
    l = e.sum(-1, keepdim=True)
    p = e / l
    o = p @ V
    live = p > 0
    # ---- score error E_s
    prods = Q[:, None, :] * K[None, :, :]                                   # (Tq, Tk, dh)
    S = prods.cumsum(-1)
    if kernel == FP32:
        es = scale * _fma_chain(S, -1) + U * x.abs()
    else:
        acc = 2 * U * (S[..., 15::16].abs().sum(-1) + prods.abs().sum(-1))
        es = scale * (_split_sum(Q[:, None, :], K[None, :, :], -1) + acc) + 2 * U * x.abs()
    del prods, S
    if M is not None:
        es = es + U * xm.abs()
    es = es + U * (xm - m).abs()
    # ---- exponentials: expf of every p, then each later rescale of the running max
    tmax = torch.stack([xm[:, t * tile:(t + 1) * tile].max(-1).values for t in range(nkt)], -1)   # (Tq, nkt)
    run = tmax.cummax(-1).values
    step = torch.zeros_like(run)
    if nkt > 1:
        prev, cur = run[:, :-1], run[:, 1:]
        step[:, 1:] = torch.where(torch.isfinite(prev), 4 * U + U * (cur - prev), torch.zeros_like(cur))
    later = step.flip(-1).cumsum(-1).flip(-1) - step                       # rescales after tile t
    tile_of_key = torch.arange(Tk) // tile
    eexp = 4 * U + later[:, tile_of_key]                                    # (Tq, Tk)
    w = torch.where(live, p * torch.where(live, es + eexp, torch.zeros_like(es)), torch.zeros_like(p))
    A = (w[:, :, None] * (V[None, :, :] - o[:, None, :]).abs()).sum(1)    # (Tq, dh)
    # ---- P V accumulation
    pv = p[:, :, None] * V[None, :, :]                                      # (Tq, Tk, dh)
    O = pv.cumsum(1)
    ends = [min((t + 1) * tile, Tk) - 1 for t in range(nkt)]
    resc = U * O[:, ends, :].abs().sum(1)
    if kernel == FP32:
        epv = _fma_chain(O, 1) + resc
    else:
        pt = e * live                                                       # the kernel's unnormalised P, in [0, 1]
        t = (pt[:, :, None] + SPLIT_FLOOR * live[:, :, None]) * (V[None, :, :].abs() + SPLIT_FLOOR)
        split = SPLIT_EPS * torch.minimum(t.sum(1), LAMBDA * t.square().sum(1).sqrt()) / l
        ks_ends = list(range(15, Tk, 16)) + ([Tk - 1] if Tk % 16 else [])
        epv = split + 2 * U * (O[:, ks_ends, :].abs().sum(1) + pv.abs().sum(1)) + resc
    del pv, O
    # ---- normalisation
    depth = (kpl - 1) + 5 + 2 * nkt + 3 if kernel == FP32 else 15 + 2 * nkt + 2 + 4
    bar = A + epv + depth * U * o.abs()
    return o, bar


def reference(q, k, v, mask, H, dh, plan):
    """fp64 o (B, Tq, D) and its per-element bar for the kernel family of `plan`"""
    scale = float(torch.tensor(1.0 / math.sqrt(dh), dtype=torch.float32))
    Q, K, V = _heads(q, H), _heads(k, H), _heads(v, H)
    B, _, Tq, _ = Q.shape
    o = torch.empty(B, H, Tq, dh, dtype=torch.float64)
    bar = torch.empty_like(o)
    for b in range(B):
        for h in range(H):
            M = mask[b, h].double() if mask is not None else None
            o[b, h], bar[b, h] = _head_ref(Q[b, h], K[b, h], V[b, h], M, scale, plan)
    return o.transpose(1, 2).reshape(B, Tq, H * dh), bar.transpose(1, 2).reshape(B, Tq, H * dh)


@functools.lru_cache(maxsize=None)
def case_reference(cid):
    c = CASE_BY_ID[cid]
    q, k, v, _, mask = inputs(cid)
    return reference(q, k, v, mask, c["H"], c["dh"], intended_plan(c))


def tf32(x):
    """round fp32 values to TF32 (10 stored mantissa bits, to nearest even)"""
    i = x.float().contiguous().view(torch.int32)
    i = (i + 0x0FFF + ((i >> 13) & 1)) & ~0x1FFF
    return i.view(torch.float32).double()


def wrong_kernel(q, k, v, mask, H, dh, rnd):
    """a kernel that rounds Q, K, V and the unnormalised P once with `rnd` and computes the rest exactly"""
    scale = float(torch.tensor(1.0 / math.sqrt(dh), dtype=torch.float32))
    Q, K, V = (rnd(_heads(t, H)) for t in (q, k, v))
    x = Q @ K.transpose(-1, -2) * scale
    if mask is not None:
        x = x + mask.double()
    e = torch.exp(x - x.max(-1, keepdim=True).values)
    o = (rnd(e) @ V) / e.sum(-1, keepdim=True)
    B, _, Tq, _ = o.shape
    return o.transpose(1, 2).reshape(B, Tq, H * dh)


WRONG = {"fp16 operands, no f16x2 correction": lambda t: t.half().double(), "TF32 operands": tf32}


# ------------------------------------------------------------------------------------------ parameters and the plan query
FAKE_BASE = 1 << 32


def params(c, addr, stored):
    """AttnParams of the case, with buffer base addresses from addr(name)"""
    _, views = _layout(c)
    p = L.AttnParams()
    for name in ("q", "k", "v", "o"):
        buf, off, sb, st = views[name]
        setattr(p, name, addr(buf) + 4 * off)
        setattr(p, name + "_sb", sb)
        setattr(p, name + "_st", st)
    if stored is not None:
        _, (sb, sh, sq), off = stored
        p.mask, p.mask_sb, p.mask_sh, p.mask_sq = addr("mask") + 4 * off, sb, sh, sq
    p.B, p.H, p.Tq, p.Tk, p.dh = c["B"], c["H"], c["Tq"], c["Tk"], c["dh"]
    p.scale = 1.0 / math.sqrt(c["dh"])
    return p


def fake_params(c):
    """made-up, 256-byte aligned addresses: the plan reads only their alignment"""
    names = sorted(_layout(c)[0]) + ["mask"]
    return params(c, lambda n: FAKE_BASE + (names.index(n) << 28), make_mask(c, key_tile(intended_plan(c)), gen(0)))


def query(p, entry, pair):
    out = (C.c_int32 * 6)()
    rc = L.lib().mtts_attention_plan_query(C.byref(p) if p is not None else None, int(entry == "tc"), pair, out)
    return rc if rc else tuple(out)


# ------------------------------------------------------------------------------------------ CPU
def _all_instantiations():
    fp32 = {(FP32, dh, rw, 8, kpl) for dh in (64, 96, 128) for rw in range(1, 9) for kpl in (1, 2)}
    fp32 |= {(FP32, 256, 4, 4, 1), (FP32, 512, 4, 4, 1)}
    return fp32 | {(TC, dh, 0, 0, 0) for dh in (64, 96, 128)} | {(PAIR, 64, 0, 0, 0), (PAIR, 96, 0, 0, 0)}


def test_case_table_reaches_every_instantiation():
    assert len(CASE_BY_ID) == len(CASES)
    reached, scalar = set(), set()
    for c in CASES:
        plan = query(fake_params(c), c["entry"], c["pair"])
        assert plan == intended_plan(c), (case_id(c), plan)
        reached.add(plan[:5])
        if not plan[5]:
            scalar.add(plan[1])
    want = _all_instantiations()
    assert reached == want, dict(missing=sorted(want - reached), extra=sorted(reached - want))
    assert len(want) == 48 + 2 + 3 + 2
    assert scalar == {64, 96, 128, 256, 512}, scalar
    # a misaligned Tq >= 65 call on the fp16-range entry point falls back from the tc kernel
    assert any(c["layout"] == "misaligned" and c["entry"] == "tc" and c["Tq"] >= 65 and c["dh"] <= 128 for c in CASES)


def test_case_table_reaches_every_axis():
    seen = set()
    for c in CASES:
        plan = intended_plan(c)
        fam = ("tc" if plan[0] != FP32 else "fp32" if c["dh"] <= 128 else "fp32-wide")
        tile = key_tile(plan)
        for a in ("mask", "layout", "mag"):
            seen.add((fam, a, c[a]))
        if c["mask"].startswith("edge") and c["Tk"] > tile:
            seen.add((fam, "first key tile masked"))
        if c["mask"].startswith("pad"):
            lens = pad_lengths(c["Tk"], tile, c["B"])
            seen.add((fam, "pad ends inside a tile", any(n % tile for n in lens if n < c["Tk"])))
            seen.add((fam, "pad ends at a tile edge", any(n % tile == 0 for n in lens if n < c["Tk"])))
        seen.add((fam, "key tiles", min(-(-c["Tk"] // tile), 3)))
        if plan[0] == FP32:
            seen.add((fam, "query CTAs > 1", -(-c["Tq"] // (plan[2] * plan[3])) > 1))
    for fam in ("fp32", "fp32-wide", "tc"):
        for kind in ("none", "causal", "pad", "pad1e9", "rand", "edge", "edge1e9"):
            assert (fam, "mask", kind) in seen, (fam, kind)
        for mag in ("randn", "peaky", "flat"):
            assert (fam, "mag", mag) in seen, (fam, mag)
        for lay in ("contig", "packed", "strided_o"):
            assert (fam, "layout", lay) in seen, (fam, lay)
        assert (fam, "first key tile masked") in seen, fam
        assert (fam, "pad ends inside a tile", True) in seen and (fam, "pad ends at a tile edge", True) in seen, fam
        assert {(fam, "key tiles", n) for n in (1, 2, 3)} <= seen, fam
    assert ("fp32", "query CTAs > 1", True) in seen and ("fp32-wide", "query CTAs > 1", True) in seen
    for fam in ("fp32", "fp32-wide"):
        assert (fam, "layout", "misaligned") in seen
    assert {c["dh"] for c in CASES if c["layout"] == "decode"} == {64, 96}
    assert {c["dh"] for c in CASES if c["layout"] == "lastrow"} == {64, 96}
    assert {c["Tq"] for c in CASES if intended_plan(c)[0] == TC} >= {65, 128, 129, 200}
    assert {c["Tk"] for c in CASES if intended_plan(c)[0] == TC} >= {1, 7, 64, 65, 300}
    assert {c["Tq"] for c in CASES if intended_plan(c)[0] == PAIR} == {16, 33, 64}
    assert {c["Tk"] for c in CASES if intended_plan(c)[:2] == (FP32, 256)} >= {1, 32, 33, 100, 257}
    assert {c["Tq"] for c in CASES if intended_plan(c)[:2] == (FP32, 512)} >= {1, 16, 17, 70}
    assert max(c["H"] for c in CASES) == 16 and min(c["B"] for c in CASES) >= 2


def _edge(**kw):
    c = _case(**dict(dict(dh=64, H=2, B=2, Tq=70, Tk=70), **kw))
    return fake_params(c)


def test_routing_edges():
    # the full-range entry point never leaves the fp32 kernel, whatever pair_min says
    for c in CASES:
        plan = query(fake_params(c), "f32", 16)
        assert plan[0] == FP32, case_id(c)
        assert plan == query(fake_params(c), "f32", OFF)
    q = query
    # Tq 64 / 65 on the fp16-range entry point
    assert q(_edge(Tq=64, Tk=64), "tc", OFF) == (FP32, 64, 8, 8, 2, 1)
    assert q(_edge(Tq=65, Tk=64), "tc", OFF) == (TC, 64, 0, 0, 0, 1)
    assert q(_edge(Tq=65, Tk=1, dh=128), "tc", OFF) == (TC, 128, 0, 0, 0, 1)
    assert q(_edge(Tq=65, Tk=65, dh=256), "tc", OFF) == (FP32, 256, 4, 4, 1, 1)
    # RW = ceil(Tq / 8), capped at 8; Tk 32 / 33 switches KPL (dh <= 128 only)
    for Tq, rw in ((1, 1), (8, 1), (9, 2), (24, 3), (25, 4), (56, 7), (57, 8), (200, 8)):
        assert q(_edge(Tq=Tq, Tk=5), "f32", OFF)[2] == rw, Tq
    assert q(_edge(Tk=32), "f32", OFF)[4] == 1 and q(_edge(Tk=33), "f32", OFF)[4] == 2
    assert q(_edge(Tk=33, dh=512, H=1), "f32", OFF) == (FP32, 512, 4, 4, 1, 1)
    # the pair route: Tq == Tk <= 64, even H, dh 64 | 96, Tq >= pair_min
    T = dict(Tq=40, Tk=40)
    assert q(_edge(**T), "tc", 40) == (PAIR, 64, 0, 0, 0, 1)
    assert q(_edge(**T, dh=96), "tc", 16) == (PAIR, 96, 0, 0, 0, 1)
    assert q(_edge(**T), "tc", 41)[0] == FP32
    assert q(_edge(**T), "tc", OFF)[0] == FP32
    assert q(_edge(Tq=40, Tk=41), "tc", 16)[0] == FP32
    assert q(_edge(**T, H=3), "tc", 16)[0] == FP32
    assert q(_edge(**T, dh=128), "tc", 16)[0] == FP32
    assert q(_edge(Tq=64, Tk=64), "tc", 16)[0] == PAIR
    assert q(_edge(Tq=65, Tk=65), "tc", 16)[0] == TC
    # alignment: a 4-byte offset q, k or v, or a row / batch stride that is not a multiple of 4 floats, takes the scalar
    # path and keeps a Tq >= 65 call off the tc kernel; an unaligned output only does the latter
    for name in ("q", "k", "v"):
        p = _edge()
        setattr(p, name, getattr(p, name) + 4)
        assert q(p, "tc", OFF) == (FP32, 64, 8, 8, 2, 0), name
        for field in (name + "_st", name + "_sb"):
            p = _edge()
            setattr(p, field, getattr(p, field) + 2)
            assert q(p, "tc", OFF) == (FP32, 64, 8, 8, 2, 0), field
    p = _edge()
    p.o += 4
    assert q(p, "tc", OFF) == (FP32, 64, 8, 8, 2, 1)
    p = _edge()
    p.o_st += 2
    assert q(p, "tc", OFF) == (FP32, 64, 8, 8, 2, 1)
    p = _edge(Tq=40, Tk=40)
    p.k += 4
    assert q(p, "tc", 16) == (FP32, 64, 5, 8, 2, 0)
    # nothing to launch, and the argument checks of the launches
    assert q(_edge(B=0), "tc", OFF)[0] == NONE and q(_edge(Tq=0), "tc", OFF)[0] == NONE
    assert q(_edge(dh=32), "f32", OFF) == UNSUPPORTED and q(_edge(dh=32), "tc", OFF) == UNSUPPORTED
    assert q(_edge(dh=32, B=0), "f32", OFF)[0] == NONE                   # B = 0 launches nothing before the dh check
    for bad in (dict(H=0), dict(Tk=0), dict(B=-1), dict(Tq=-1), dict(H=65536)):
        assert q(_edge(**bad), "tc", OFF) == BAD_ARG, bad
    p = _edge()
    p.q = None
    assert q(p, "tc", OFF) == BAD_ARG
    p = _edge()
    p.o_planes, p.o_planes_ld, p.o_plane_stride = FAKE_BASE, 130, 4096
    assert q(p, "tc", OFF) == BAD_ARG
    assert q(None, "tc", OFF) == BAD_ARG


def test_bar_rejects_plausible_wrong_kernels():
    """The tc kernel without its f16x2 correction terms and the fp32 kernel on TF32 operands exceed every case's bar by at
    least 4x wherever they differ from fp64."""
    worst = {name: (math.inf, None) for name in WRONG}
    for c in CASES:
        cid = case_id(c)
        q, k, v, _, mask = inputs(cid)
        ref, bar = case_reference(cid)
        for name, rnd in WRONG.items():
            err = (wrong_kernel(q, k, v, mask, c["H"], c["dh"], rnd) - ref).abs()
            if err.max().item() == 0:
                continue
            r = (err / bar).max().item()
            assert r >= 4, (cid, name, r)
            worst[name] = min(worst[name], (r, cid))
    for name, (r, cid) in worst.items():
        print(f"{name}: at least {r:.1f}x the bar (smallest at {cid})")


# ------------------------------------------------------------------------------------------ GPU
def _bits(t):
    return t.contiguous().view(torch.int16).cpu()


class _Launch:
    """device buffers of a case laid out as the case says, and its launches"""

    def __init__(self, c):
        cid = case_id(c)
        self.c = c
        q, k, v, stored, _ = inputs(cid)
        bufs, views = _layout(c)
        g = gen(zlib.crc32(cid.encode()) + 1)
        self.buf = {n: torch.randn(size, generator=g).to(DEV) for n, size in bufs.items()}   # unread parts: garbage
        for name, t in (("q", q), ("k", k), ("v", v)):
            buf, off, sb, st = views[name]
            torch.as_strided(self.buf[buf], t.shape, (sb, st, 1), off).copy_(t.to(DEV))
        self.buf["o"].fill_(7.0)
        if stored is not None:
            self.buf["mask"] = stored[0].reshape(-1).to(DEV)
        self.p = params(c, lambda n: self.buf[n].data_ptr(), stored)
        self.fn = L.lib().mtts_attention_tc_f32 if c["entry"] == "tc" else L.lib().mtts_attention_f32
        _, off, sb, st = views["o"]
        self.o_view = (off, sb, st)

    def out(self, o_buf):
        c = self.c
        off, sb, st = self.o_view
        D = c["H"] * c["dh"]
        return torch.as_strided(o_buf, (c["B"], c["Tq"], D), (sb, st, 1), off).cpu()

    def run(self, p=None, o_buf=None):
        from megatts2_b200 import ops
        p = p or self.p
        if o_buf is not None:
            p = _copy(p)
            p.o = o_buf.data_ptr() + 4 * self.o_view[0]
        L.check(self.fn(C.byref(p), ops._stream()))
        torch.cuda.synchronize()


def _copy(p):
    q = L.AttnParams()
    C.pointer(q)[0] = p
    return q


@gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_attention_vs_fp64(c):
    from megatts2_b200 import ops
    dev = torch.device(DEV)
    cid = case_id(c)
    B, Tq, D = c["B"], c["Tq"], c["H"] * c["dh"]
    ref, bar = case_reference(cid)
    run = _Launch(c)
    plan = query(run.p, c["entry"], c["pair"])
    assert plan == intended_plan(c), (plan, intended_plan(c))
    ops.tc_overflow(dev)                                            # binds and clears the range flag
    prev = ops.set_attention_pair_min(c["pair"])
    try:
        o_buf = run.buf["o"]
        run.run()
        o = run.out(o_buf)
        # a repeat launch is bit-identical
        again = torch.full_like(o_buf, 7.0)
        run.run(o_buf=again)
        assert torch.equal(run.out(again), o), "a repeat launch differs"
        # the last item of the batch, launched alone
        b = B - 1
        p1 = _copy(run.p)
        p1.B = 1
        for name in ("q", "k", "v"):
            setattr(p1, name, getattr(p1, name) + 4 * b * getattr(p1, name + "_sb"))
        if p1.mask:
            p1.mask += 4 * b * p1.mask_sb
        one = torch.full_like(o_buf, 7.0)
        p1.o = one.data_ptr() + 4 * (run.o_view[0] + b * run.o_view[1])
        assert query(p1, c["entry"], c["pair"]) == plan
        run.run(p1)
        assert torch.equal(run.out(one)[b], o[b]), "item b of the batch differs from a single-item launch"
        # operand planes for the out-projection GEMM, from the same launch as fp32 rows
        for fmt in (pack.FMT_BF16X3, pack.FMT_F16X2):
            npl = 3 - fmt
            planes = torch.full((npl, B * Tq, D), 7.0, dtype=pack.plane_dtype(fmt), device=DEV)
            pp = _copy(run.p)
            pp.o_planes, pp.o_plane_stride, pp.o_planes_ld, pp.o_planes_fmt = planes.data_ptr(), B * Tq * D, D, fmt
            ob = torch.full_like(o_buf, 7.0)
            run.run(pp, o_buf=ob)
            assert torch.equal(run.out(ob), o), "the launch with a plane output stores different fp32 rows"
            spec = pack.pack_tc_planes(o.reshape(B * Tq, D), fmt)
            assert torch.equal(_bits(planes), _bits(spec)), f"plane output ({fmt}) differs from pack_tc_planes"
    finally:
        ops.set_attention_pair_min(0 if prev >= (1 << 30) else prev)
    if plan[0] != FP32:
        assert not ops.tc_overflow(dev), "the range flag was raised by in-range operands"
    if c["layout"] == "strided_o":
        pad = o_buf.view(B, Tq, D + 32)[..., D:]
        assert bool((pad == 7.0).all()), "columns past D of the strided output were written"
    err = (o.double() - ref).abs()
    ratio = (err / bar).max().item()
    print(f"{cid}: {plan_str(plan)}  error / bar {ratio:.3f}")
    helpers.record("attention_oracle", dict(case=cid, kernel=KNAME[plan[0]], plan=list(plan), err_to_bound=ratio,
                                            max_err=err.max().item()))
    if not ratio <= 1:
        i = int((err / bar).argmax())
        bb, t, d = i // (Tq * D), (i // D) % Tq, i % D
        pytest.fail(f"error {err.max().item():.3e} is {ratio:.2f}x the bound; worst at b={bb} t={t} d={d} "
                    f"(|err| {err[bb, t, d].item():.3e}, bound {bar[bb, t, d].item():.3e})")
