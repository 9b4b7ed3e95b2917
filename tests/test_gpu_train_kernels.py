"""GPU: the training kernels (csrc/train.cu) and the autograd Functions (megatts2_b200/autograd.py) against fp64, one at a
time, with dropout on.

Every reference is plain torch fp64 on the CPU over the exact fp32 values the kernel received.  Where a rigorous fp32
error bound exists the test asserts it (u = 2^-24; an fp32 sum whose every term passes through at most d roundings is
within d * u * sum|terms| of the exact sum, up to second-order terms the small margins below cover):
  bmm            |C - C*| <= (K + 2) u (|alpha| |A| @ |B| + |C0|)                  (K FMAs, the alpha scale, the += of C0)
  softmax_bwd    |dS - dS*| <= (ceil(Tk / 32) + 9) u P (|dP| + sum |dP| P)         (lane FMA chain + 5 shuffle levels)
  colsum         |out - out*| <= (rows + 2) u (sum |in| + |out0|)
  embedding_bwd  |dW - dW*| <= n u sum |dy|      (n = how often the row's id occurs: the atomics add in any order)
  rowdot         |out - out*| <= (ceil(C / 32) + 6) u sum |a b|
  relu_bwd       exact
Everywhere else (softmax_fwd, layernorm_bwd, the Functions) the bar is about ten times the error measured on an H100
80GB HBM3 at a 400 W power limit; each test records what it measured through helpers.record ($MEGATTS2_PARITY_LOG).

Dropout: the Functions draw their masks from ``torch.rand``.  The tests wrap it to record the draws, and the fp64 reference
applies the product's own keep tensor, keep = (draw >= p) / (1 - p) in fp32, so a dropped, doubled or misplaced keep
factor anywhere in the forward or the backward shows up as an error of order p."""
import contextlib
import math

import pytest
import torch
import torch.nn.functional as F

import helpers
from megatts2_b200 import _lib as L
from megatts2_b200 import autograd as A
from megatts2_b200 import ops, pack
from megatts2_b200.utils.utils import make_attn_mask
from oracle import ref_megatts2 as R

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
DEV = "cuda"
U = 2.0 ** -24
F32_EPS_1E5 = float(torch.tensor(1e-5, dtype=torch.float32))      # the eps the kernels see

# measured-error bars: about 10x the largest error measured on an H100 80GB HBM3, 400 W (measured value in the comment)
SOFTMAX_FWD_ULPS = 200.0         # |P - P*| / P*, in units of u                                         (19.7)
LN_BWD_DX_ULPS = 40.0            # |dx - dx*| / (rstd max|dy gamma|), per row, in units of u            (3.6)
LN_BWD_DGAMMA_ULPS = 25.0        # |dgamma - dgamma*| / sum_r |dy| (1 + |xhat|), in units of u          (2.3)
LN_BWD_OFFSET_DX = 3e-4          # the row with mean 1e4: the same two measures, not in units of u      (3.0e-5)
LN_BWD_OFFSET_DGAMMA = 2e-3      #                                                                      (1.9e-4)
ATTN_REL = 1e-5                  # max |got - ref| / max |ref| of out, dq, dk, dv                       (9.9e-7)
LINEAR_REL = 6e-6                # y, dx, dw, db                                                        (5.9e-7)
LAYERNORM_FN_REL = 2e-6          # y, dx, dgamma, dbeta                                                 (1.8e-7)
LAYER_REL = 1e-5                 # y, dx and every parameter gradient of one encoder layer, dropout 0.1 (1.1e-6)
LAYER_KEY_BIAS = 1e-4            # the key bias' gradient, zero in exact arithmetic (see the test)      (1.1e-5)


def gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


def _lib():
    return L.lib()


def _rel(got, ref, floor=0.0):
    """max |got - ref| / max(max |ref|, floor), fp64"""
    got = got.detach().double().cpu()
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), floor, 1e-300)


def _within(err, bound):
    """every |error| within its rigorous bound; returns the largest error / bound (0 where both are 0)"""
    assert bool((err <= bound).all()), f"error above the fp32 bound: worst excess {(err - bound).max().item():.3e}"
    nz = bound > 0
    return (err[nz] / bound[nz]).max().item() if bool(nz.any()) else 0.0


class _Draws:
    """records every torch.rand draw made inside ``with draws:`` (the dropout masks of the Functions)"""

    def __init__(self, monkeypatch):
        self.mp, self.draws = monkeypatch, []

    def __enter__(self):
        real = torch.rand

        def rand(*a, **k):
            r = real(*a, **k)
            self.draws.append(r)
            return r
        self.ctx = self.mp.context()
        self.ctx.__enter__().setattr(torch, "rand", rand)
        return self

    def __exit__(self, *exc):
        self.ctx.__exit__(*exc)
        return False


def _keep(draw, p):
    """nn.Dropout's keep tensor for a recorded draw, the fp32 values the product multiplies by, as fp64 on the CPU"""
    return ((draw >= p).to(torch.float32) / (1.0 - p)).double().cpu()


# ------------------------------------------------------------------------------------------ bmm
SIZES = (1, 15, 16, 17, 63, 64, 65, 200)


def _head_view(Z1, Z2, R_, Cc, cols_fast, g, pad=0):
    """(Z1, Z2, R_, Cc) fp32 CUDA view into a (B, T, H, d)-shaped buffer (the head layout: z1 = b, z2 = h), with either
    the column index (d = Cc) or the row index (d = R_) unit-stride.  Returns (base, view)."""
    if cols_fast:
        base = torch.randn(Z1, R_, Z2, Cc + pad, generator=g).to(DEV)
        return base, base[..., :Cc].permute(0, 2, 1, 3)
    base = torch.randn(Z1, Cc, Z2, R_ + pad, generator=g).to(DEV)
    return base, base[..., :R_].permute(0, 2, 3, 1)


def _bmm(a, sa, b, sb, c, sc, Z1, Z2, M, N, K, alpha=1.0, accumulate=0):
    L.check(_lib().mtts_bmm_f32(ops._ptr(a), *sa, ops._ptr(b), *sb, ops._ptr(c), *sc, Z1, Z2, M, N, K, alpha,
                                accumulate, ops._stream()))


@pytest.mark.parametrize("a_fast,b_fast", [("k", "n"), ("m", "n"), ("k", "k"), ("m", "k")])
def test_bmm_layouts_and_tails_within_fp32_bound(a_fast, b_fast):
    """Every (M, K) pair of SIZES, with N running through SIZES too, on (B, T, H, dh) head views: each 64 x 64 tile and
    each 16-wide k slice has tails.  alpha != 1 and accumulate = 1 on a preloaded C alternate over the cases; the padding
    columns of C stay untouched."""
    g = gen(101 + 7 * ("mk".index(a_fast)) + ("nk".index(b_fast)))
    Z1, Z2 = 2, 3
    worst = 0.0
    li = ("mk".index(a_fast)) * 2 + ("nk".index(b_fast))
    for i, M in enumerate(SIZES):
        for j, K in enumerate(SIZES):
            N = SIZES[(i + 3 * j + li) % len(SIZES)]
            idx = i * len(SIZES) + j
            alpha = float(torch.tensor((1.0, -0.37, 0.125)[idx % 3], dtype=torch.float32))
            acc = idx % 2
            _, a = _head_view(Z1, Z2, M, K, a_fast == "k", g)
            _, b = _head_view(Z1, Z2, K, N, b_fast == "n", g)
            cbase, c = _head_view(Z1, Z2, M, N, True, g, pad=3)
            c0 = c.double().cpu()
            pad0 = cbase[..., N:].clone()
            _bmm(a, a.stride(), b, b.stride(), c, c.stride(), Z1, Z2, M, N, K, alpha, acc)
            a64, b64 = a.double().cpu(), b.double().cpu()
            ref = alpha * (a64 @ b64) + (c0 if acc else 0.0)
            bound = (K + 2) * U * (abs(alpha) * (a64.abs() @ b64.abs()) + (c0.abs() if acc else 0.0))
            ratio = _within((c.double().cpu() - ref).abs(), bound)
            worst = max(worst, ratio)
            assert torch.equal(cbase[..., N:], pad0), f"bmm wrote outside C at M={M} N={N} K={K}"
    helpers.record("train_bmm", dict(a_fast=a_fast, b_fast=b_fast, cases=len(SIZES) ** 2, worst_err_over_bound=worst))


def test_bmm_empty_products_and_grid_refusals():
    g = gen(111)
    a = torch.randn(2, 3, 17, 5, generator=g).to(DEV)
    b = torch.randn(2, 3, 5, 19, generator=g).to(DEV)
    for M, N, K in ((0, 19, 5), (17, 0, 5), (17, 19, 0)):
        for acc in (0, 1):
            c = torch.randn(2, 3, 17, 19, generator=g).to(DEV)
            c0 = c.clone()
            _bmm(a, a.stride(), b, b.stride(), c, c.stride(), 2, 3, M, N, K, -0.5, acc)
            if K == 0 and not acc:
                assert bool((c == 0).all()), "K = 0 writes alpha * (empty sum) = 0"
            else:
                assert torch.equal(c, c0), f"M={M} N={N} K={K} accumulate={acc} must leave C unchanged"
    c = torch.randn(2, 3, 17, 19, generator=g).to(DEV)
    c0 = c.clone()
    with pytest.raises(L.MttsError, match="grid"):
        _bmm(a, (0,) * 4, b, (0,) * 4, c, (0,) * 4, 256, 257, 1, 1, 1)          # Z1 * Z2 = 65792 > 65535
    with pytest.raises(L.MttsError, match="grid"):
        _bmm(a, (0,) * 4, b, (0,) * 4, c, (0,) * 4, 1, 1, 64 * 65535 + 1, 1, 1)  # ceil(M / 64) = 65536
    torch.cuda.synchronize()
    assert torch.equal(c, c0)


# ------------------------------------------------------------------------------------------ softmax
TKS = (1, 5, 31, 32, 33, 64, 65, 257)


def _rand_mask(shape, g):
    """additive mask: -inf with probability 0.3, else uniform in [-3, 3]; one random entry of each row is finite"""
    m = torch.empty(shape).uniform_(-3, 3, generator=g)
    m[torch.rand(shape, generator=g) < 0.3] = float("-inf")
    m.scatter_(-1, torch.randint(0, shape[-1], shape[:-1] + (1,), generator=g), 0.0)
    return m


def _softmax_fwd(S, mask, B, H, Tq, Tk, keep, P, Pd):
    sb, sh, sq = mask.stride()[:3] if mask is not None else (0, 0, 0)
    L.check(_lib().mtts_softmax_fwd_f32(ops._ptr(S), ops._ptr(mask), sb, sh, sq, B, H, Tq, Tk, ops._ptr(keep), ops._ptr(P),
                                        ops._ptr(Pd), ops._stream()))


def _prob_ulps(got, ref):
    """largest |got - ref| / ref in units of u; got must be exactly 0 wherever ref is"""
    got = got.double().cpu()
    pos = ref > 0
    assert bool((got[~pos] == 0).all()), "a probability that is exactly 0 (masked or dropped) came out nonzero"
    return ((got - ref).abs()[pos] / ref[pos]).max().item() / U


@pytest.mark.parametrize("Tk", TKS)
def test_softmax_fwd_masks_and_keep_vs_fp64(Tk):
    """30 rows (B 2, H 3, Tq 5: not a multiple of the kernel's 8 rows per CTA); masks broadcast along b, h and q by zero
    strides; with a keep tensor both P and Pd = P * keep; without one, Pd aliasing P and Pd a separate buffer."""
    g = gen(200 + Tk)
    B, H, Tq = 2, 3, 5
    S = (torch.randn(B, H, Tq, Tk, generator=g) * 2).to(DEV)
    p = 0.1
    keep = ((torch.rand(B, H, Tq, Tk, generator=g) >= p).float() / (1 - p)).to(DEV)
    worst = 0.0
    for shape in (None, (B, 1, 1, Tk), (1, H, 1, Tk), (1, 1, Tq, Tk), (B, H, Tq, Tk)):
        m = _rand_mask(shape, g).to(DEV).expand(B, H, Tq, Tk) if shape else None
        ref = torch.softmax(S.double().cpu() + (m.double().cpu() if m is not None else 0.0), -1)
        P, Pd = torch.full_like(S, float("nan")), torch.full_like(S, float("nan"))
        _softmax_fwd(S, m, B, H, Tq, Tk, keep, P, Pd)
        worst = max(worst, _prob_ulps(P, ref), _prob_ulps(Pd, ref * keep.double().cpu()))
        P2 = torch.full_like(S, float("nan"))
        _softmax_fwd(S, m, B, H, Tq, Tk, None, P2, P2)                           # Pd aliases P
        assert torch.equal(P2, P), "the result without keep equals P of the run with keep"
        Pd2 = torch.full_like(S, float("nan"))
        _softmax_fwd(S, m, B, H, Tq, Tk, None, P2, Pd2)                          # separate Pd, no keep: Pd = P
        assert torch.equal(Pd2, P)
    helpers.record("train_softmax_fwd", dict(Tk=Tk, worst_ulps=worst, bar=SOFTMAX_FWD_ULPS))
    assert worst <= SOFTMAX_FWD_ULPS, f"softmax_fwd error {worst:.1f} u"


def test_softmax_fwd_fully_masked_row_is_nan_like_torch():
    B, H, Tq, Tk = 1, 2, 3, 40
    S = torch.randn(B, H, Tq, Tk, generator=gen(230))
    m = torch.zeros(B, H, Tq, Tk)
    m[0, 1, 2] = float("-inf")
    ref = torch.softmax(S.double() + m.double(), -1)
    assert bool(ref[0, 1, 2].isnan().all())                                      # torch's convention
    P = torch.zeros(B, H, Tq, Tk, device=DEV)
    _softmax_fwd(S.to(DEV), m.to(DEV), B, H, Tq, Tk, None, P, P)
    P = P.cpu()
    assert bool(P[0, 1, 2].isnan().all()), "a fully masked row is NaN, as in torch.softmax"
    ok = ~ref.isnan()
    assert bool(torch.isfinite(P[ok]).all()) and (P.double()[ok] - ref[ok]).abs().max().item() < SOFTMAX_FWD_ULPS * U


@pytest.mark.parametrize("Tk", TKS)
def test_softmax_bwd_with_and_without_keep_within_fp32_bound(Tk):
    """dS = P (dP - <dP, P>), dP = dPd * keep, on probabilities with exact zeros (masked keys)"""
    g = gen(300 + Tk)
    rows = 30
    P = torch.softmax(torch.randn(rows, Tk, generator=g) * 2 + _rand_mask((rows, Tk), g), -1)
    dPd = torch.randn(rows, Tk, generator=g)
    keep = (torch.rand(rows, Tk, generator=g) >= 0.1).float() / 0.9
    worst = 0.0
    for kp in (None, keep):
        dS = torch.full((rows, Tk), float("nan"), device=DEV)
        Pg, dPdg = P.to(DEV), dPd.to(DEV)
        kg = kp.to(DEV) if kp is not None else None
        L.check(_lib().mtts_softmax_bwd_f32(ops._ptr(Pg), ops._ptr(dPdg), ops._ptr(kg), ops._ptr(dS), Tk, rows, ops._stream()))
        P64, dP = P.double(), dPd.double() * (kp.double() if kp is not None else 1.0)
        t = (dP * P64).sum(-1, keepdim=True)
        ref = P64 * (dP - t)
        bound = (math.ceil(Tk / 32) + 9) * U * P64 * (dP.abs() + (dP.abs() * P64).sum(-1, keepdim=True))
        worst = max(worst, _within((dS.double().cpu() - ref).abs(), bound))
    helpers.record("train_softmax_bwd", dict(Tk=Tk, worst_err_over_bound=worst))


# ------------------------------------------------------------------------------------------ LayerNorm backward
def _ln_bwd(x, gamma, dy, C):
    rows = x.shape[0]
    nb = (rows + 7) // 8
    dx = torch.full_like(x, float("nan"))
    partial = torch.full((nb, 2, C), float("nan"), device=DEV)
    L.check(_lib().mtts_layernorm_bwd_f32(ops._ptr(x), ops._ptr(gamma), ops._ptr(dy), ops._ptr(dx), ops._ptr(partial), rows,
                                          C, 1e-5, ops._stream()))
    dgb = torch.full((2 * C,), float("nan"), device=DEV)
    L.check(_lib().mtts_colsum_f32(ops._ptr(partial), 2 * C, nb, 2 * C, ops._ptr(dgb), 0, ops._stream()))
    return dx, dgb[:C], dgb[C:], nb


def _ln_ref(x, gamma, dy):
    x64 = x.double().cpu().requires_grad_(True)
    g64 = gamma.double().cpu().requires_grad_(True)
    b64 = torch.zeros_like(g64, requires_grad=True)
    F.layer_norm(x64, (x.shape[1],), g64, b64, F32_EPS_1E5).backward(dy.double().cpu())
    xd = x64.detach()
    mean = xd.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + F32_EPS_1E5)
    return x64.grad, g64.grad, b64.grad, (xd - mean) * rstd, rstd


def _ln_errors(x, gamma, dy, C):
    """(dx error per row in units of u * rstd * max|dy gamma|, d-gamma error in units of u * sum_r |dy| (1 + |xhat|)),
    d-beta within its bound (8 warps + colsum over nb CTAs, (nb + 11) roundings)"""
    dx, dg, db, nb = _ln_bwd(x, gamma, dy, C)
    rdx, rdg, rdb, xh, rstd = _ln_ref(x, gamma, dy)
    dy64 = dy.double().cpu()
    gsc = (dy64 * gamma.double().cpu()).abs().amax(1, keepdim=True) * rstd
    e_dx = ((dx.double().cpu() - rdx).abs() / gsc).max().item() / U
    e_dg = ((dg.double().cpu() - rdg).abs() / (dy64.abs() * (1 + xh.abs())).sum(0)).max().item() / U
    _within((db.double().cpu() - rdb).abs(), (nb + 11) * U * dy64.abs().sum(0))
    return e_dx, e_dg


@pytest.mark.parametrize("C", [1, 32, 100, 384, 768, 769, 1024, 3072])
def test_layernorm_bwd_and_colsum_vs_fp64_autograd(C):
    """C = 768 needs exactly 48 KB of shared memory, 769 is the first size above it (the large-shared-memory attribute),
    3072 the limit; 333 rows leave the last CTA with 5 live warps and 3 zero-filled ones.  One row is constant (variance
    0: eps decides rstd)."""
    g = gen(400 + C)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(DEV)
    worst_dx = worst_dg = 0.0
    for rows in (1, 7, 8, 9, 333):
        x = torch.randn(rows, C, generator=g) * (0.5 + 1.5 * torch.rand(rows, 1, generator=g)) + \
            0.5 * torch.randn(rows, 1, generator=g)
        if rows >= 7:
            x[rows // 2] = 0.75
        dy = torch.randn(rows, C, generator=g)
        e_dx, e_dg = _ln_errors(x.to(DEV), gamma, dy.to(DEV), C)
        worst_dx, worst_dg = max(worst_dx, e_dx), max(worst_dg, e_dg)
    helpers.record("train_layernorm_bwd", dict(C=C, dx_ulps=worst_dx, dgamma_ulps=worst_dg))
    assert worst_dx <= LN_BWD_DX_ULPS, f"layernorm_bwd dx error {worst_dx:.1f} u"
    assert worst_dg <= LN_BWD_DGAMMA_ULPS, f"layernorm_bwd d-gamma error {worst_dg:.1f} u"


@pytest.mark.parametrize("C", [100, 768, 1024, 3072])
def test_layernorm_bwd_row_with_large_mean(C):
    """A row with mean 1e4 and unit spread: its fp32 mean carries an absolute error of up to about an ulp of 1e4 (1e-3),
    which every xhat of the row inherits - a separate, looser bar than the other rows'."""
    g = gen(450 + C)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(DEV)
    x = torch.randn(9, C, generator=g)
    x[4] += 1e4
    e_dx, e_dg = _ln_errors(x.to(DEV), gamma, torch.randn(9, C, generator=g).to(DEV), C)
    helpers.record("train_layernorm_bwd_offset_row", dict(C=C, dx_rel=e_dx * U, dgamma_rel=e_dg * U))
    assert e_dx * U <= LN_BWD_OFFSET_DX and e_dg * U <= LN_BWD_OFFSET_DGAMMA, (e_dx * U, e_dg * U)


def test_layernorm_bwd_refuses_more_than_3072_channels():
    x = torch.zeros(8, 3073, device=DEV)
    gamma = torch.ones(3073, device=DEV)
    partial = torch.zeros(1, 2, 3073, device=DEV)
    with pytest.raises(L.MttsError, match="3072"):
        L.check(_lib().mtts_layernorm_bwd_f32(ops._ptr(x), ops._ptr(gamma), ops._ptr(x), ops._ptr(x), ops._ptr(partial), 8,
                                              3073, 1e-5, ops._stream()))


# ------------------------------------------------------------------------------------------ small kernels
@pytest.mark.parametrize("C", [1, 100, 300])
def test_colsum_accumulate_leading_dimension_and_empty_within_fp32_bound(C):
    g = gen(500 + C)
    ld = C + 5
    worst = 0.0
    for rows in (0, 1, 3, 4, 5, 7, 8, 1001):
        x = torch.randn(max(rows, 1), ld, generator=g)
        for acc in (0, 1):
            out0 = torch.randn(C + 3, generator=g)
            xd, out = x.to(DEV), out0.to(DEV)
            L.check(_lib().mtts_colsum_f32(ops._ptr(xd), ld, rows, C, ops._ptr(out), acc, ops._stream()))
            out = out.cpu()
            x64 = x[:rows, :C].double()
            ref = x64.sum(0) + (out0[:C].double() if acc else 0.0)
            bound = (rows + 2) * U * (x64.abs().sum(0) + (out0[:C].double().abs() if acc else 0.0))
            worst = max(worst, _within((out[:C].double() - ref).abs(), bound))
            assert torch.equal(out[C:], out0[C:]), "colsum wrote past C"
            if rows == 0:
                assert torch.equal(out[:C], out0[:C] if acc else torch.zeros(C))
    helpers.record("train_colsum", dict(C=C, worst_err_over_bound=worst))


def test_relu_bwd_signed_zero_and_tiny_outputs():
    special = torch.tensor([0.0, -0.0, 1e-45, 1e-40, 1.1754944e-38, -1e-45, -1e-40, 1.0, -1.0, float("inf"), float("-inf")])
    g = gen(600)
    y = torch.cat([special, torch.randn(1000, generator=g), special])            # n = 1022: a partial last block
    dy = torch.randn(y.numel(), generator=g)
    yd, dyd = y.to(DEV), dy.to(DEV)
    dx = torch.full_like(yd, float("nan"))
    L.check(_lib().mtts_relu_bwd_f32(ops._ptr(yd), ops._ptr(dyd), ops._ptr(dx), y.numel(), ops._stream()))
    ref = torch.where(y > 0, dy, torch.zeros(()))
    assert torch.equal(dx.cpu(), ref), "dx = dy exactly where y > 0 (+0 and -0 are not), else 0"
    assert (special > 0).nonzero().flatten().tolist() == [2, 3, 4, 7, 9]         # the subnormals count as positive


def test_embedding_bwd_heavily_repeated_ids_within_fp32_bound():
    g = gen(700)
    V, D, rows = 40, 77, 6000
    ids = torch.randint(0, V, (rows,), generator=g)
    ids[torch.rand(rows, generator=g) < 0.9] = 7                                 # ~5400 hits on one row
    dy = torch.randn(rows, D, generator=g)
    idsd, dyd = ids.to(DEV), dy.to(DEV)
    dW = torch.zeros(V, D, device=DEV)
    L.check(_lib().mtts_embedding_bwd_f32(ops._ptr(idsd), ops._ptr(dyd), rows, D, V, ops._ptr(dW), ops._stream()))
    ref = torch.zeros(V, D, dtype=torch.float64).index_add_(0, ids, dy.double())
    mag = torch.zeros(V, D, dtype=torch.float64).index_add_(0, ids, dy.double().abs())
    n = torch.bincount(ids, minlength=V).double()[:, None]
    assert int(n.max()) > 5000
    worst = _within((dW.double().cpu() - ref).abs(), n * U * mag)
    helpers.record("train_embedding_bwd", dict(rows=rows, max_hits=int(n.max()), worst_err_over_bound=worst))


@pytest.mark.parametrize("C", [1, 31, 32, 33, 1024])
def test_rowdot_period_shorter_than_rows_within_fp32_bound(C):
    g = gen(800 + C)
    rows, period = 301, 37
    a, b = torch.randn(rows, C, generator=g), torch.randn(period, C, generator=g)
    ad, bd = a.to(DEV), b.to(DEV)
    out = torch.full((rows,), float("nan"), device=DEV)
    L.check(_lib().mtts_rowdot_f32(ops._ptr(ad), ops._ptr(bd), rows, C, period, ops._ptr(out), ops._stream()))
    bt = b.double()[torch.arange(rows) % period]
    ref = (a.double() * bt).sum(1)
    bound = (math.ceil(C / 32) + 6) * U * (a.double() * bt).abs().sum(1)
    worst = _within((out.double().cpu() - ref).abs(), bound)
    helpers.record("train_rowdot", dict(C=C, worst_err_over_bound=worst))


# ------------------------------------------------------------------------------------------ AttentionFn
def _attention_ref(q, k, v, H, mask, keep, go):
    """fp64 autograd of (softmax(Q K^T / sqrt(dh) + mask) * keep) V"""
    q, k, v = (t.detach().double().cpu().requires_grad_(True) for t in (q, k, v))
    B, Tq, D = q.shape
    Tk, dh = k.shape[1], D // H
    qh = q.view(B, Tq, H, dh).transpose(1, 2)
    kh, vh = (t.view(B, Tk, H, dh).transpose(1, 2) for t in (k, v))
    s = qh @ kh.transpose(-1, -2) / math.sqrt(dh)
    if mask is not None:
        s = s + mask.double().cpu()
    p = torch.softmax(s, -1)
    if keep is not None:
        p = p * keep
    out = (p @ vh).transpose(1, 2).reshape(B, Tq, D)
    out.backward(go)
    return out.detach(), q.grad, k.grad, v.grad


def _attention_case(monkeypatch, g, B, H, dh, Tq, Tk, mask, p_drop):
    D = H * dh
    q = torch.randn(B, Tq, D, generator=g).to(DEV).requires_grad_(True)
    k = torch.randn(B, Tk, D, generator=g).to(DEV).requires_grad_(True)
    v = torch.randn(B, Tk, D, generator=g).to(DEV).requires_grad_(True)
    go = torch.randn(B, Tq, D, generator=g).double()
    with _Draws(monkeypatch) as rec:
        out = A.AttentionFn.apply(q, k, v, H, mask, p_drop)
    keep = None
    if p_drop > 0:
        assert [tuple(d.shape) for d in rec.draws] == [(B, H, Tq, Tk)]
        keep = _keep(rec.draws[0], p_drop)
    else:
        assert rec.draws == []
    out.backward(go.float().to(DEV))
    refs = _attention_ref(q, k, v, H, mask, keep, go)
    # with one key (T = 1) softmax's gradient, and so dq and dk, are zero in exact arithmetic; the kernels leave a residual
    # of the order of an ulp of dP there.  Errors are taken relative to at least 0.1 of the case's largest reference entry.
    floor = 0.1 * max(r.abs().max().item() for r in refs)
    return max(_rel(got, r, floor) for got, r in zip((out, q.grad, k.grad, v.grad), refs))


@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("mask_kind", ["none", "pad", "causal+pad"])
@pytest.mark.parametrize("dh", [64, 96])
def test_attention_fn_vs_fp64_autograd(monkeypatch, dh, mask_kind, p_drop):
    """Tq = Tk in {1, 37, 64, 65, 130} at the PLM (dh 64) and ADM (dh 96) head widths; masks from make_attn_mask"""
    g = gen(900 + dh + 10 * len(mask_kind) + int(100 * p_drop))
    B, H = 2, 3
    worst = 0.0
    for T in (1, 37, 64, 65, 130):
        lens = torch.tensor([T, max(T - 5, 1)], dtype=torch.int32)
        mask = None if mask_kind == "none" else make_attn_mask(lens, H, causal=mask_kind == "causal+pad").to(DEV)
        worst = max(worst, _attention_case(monkeypatch, g, B, H, dh, T, T, mask, p_drop))
    helpers.record("train_attention_fn", dict(dh=dh, mask=mask_kind, p_drop=p_drop, worst_rel=worst, bar=ATTN_REL))
    assert worst <= ATTN_REL, f"AttentionFn relative error {worst:.3e}"


@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("dh", [64, 96])
def test_attention_fn_cross_lengths_vs_fp64_autograd(monkeypatch, dh, p_drop):
    """Tq != Tk both ways, padded keys"""
    g = gen(950 + dh + int(100 * p_drop))
    B, H = 2, 3
    worst = 0.0
    for Tq, Tk in ((37, 65), (130, 17)):
        mask = make_attn_mask(torch.tensor([Tk, Tk - 6], dtype=torch.int32), H).to(DEV)     # (B, H, 1, Tk)
        worst = max(worst, _attention_case(monkeypatch, g, B, H, dh, Tq, Tk, mask, p_drop))
    helpers.record("train_attention_fn_cross", dict(dh=dh, p_drop=p_drop, worst_rel=worst, bar=ATTN_REL))
    assert worst <= ATTN_REL, f"AttentionFn relative error {worst:.3e}"


# ------------------------------------------------------------------------------------------ LinearFn / LayerNormFn
def _relu_from_product(z_ref, y_prod):
    """The ReLU sub-gradient mask the product took (y > 0), after checking it agrees with the sign of the fp64
    pre-activation everywhere but within rounding of the kink, where either choice is right."""
    on = y_prod.detach().cpu() > 0
    clear = z_ref.abs() > 1e-4 * z_ref.abs().max()
    assert torch.equal(on[clear], (z_ref > 0)[clear]), "ReLU decided against the sign of its input"
    return on.double()


@pytest.mark.parametrize("engine", ["default", "ffma"])
@pytest.mark.parametrize("M", [1, 127, 128, 256, 300])
def test_linear_fn_both_routes_vs_fp64_autograd(M, engine):
    """M >= 128 runs the products on the tensor-core tap-GEMM under the default engine (bf16x3 operands); M = 300 has a
    dW product with a ragged row count (bmm); M < 128 and every product under FFMA take the fp32 batched matmul."""
    K, N = 192, 160
    g = gen(1000 + M)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g)
    gy = torch.randn(M, N, generator=g).double()
    worst = 0.0
    with pack.engine_scope(pack.ENGINE_FFMA) if engine == "ffma" else contextlib.nullcontext():
        assert A._tc_ok(M, K, N) == (pack.default_engine() != pack.ENGINE_FFMA and M >= 128)
        for relu in (False, True):
            for has_bias in (False, True):
                xd, wd = x.to(DEV).requires_grad_(True), w.to(DEV).requires_grad_(True)
                bd = b.to(DEV).requires_grad_(True) if has_bias else None
                y = A.linear(xd, wd, bd, relu=relu)
                y.backward(gy.float().to(DEV))
                x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
                b64 = b.double().requires_grad_(True) if has_bias else None
                z = F.linear(x64, w64, b64)
                ref = z * _relu_from_product(z.detach(), y) if relu else z
                ref.backward(gy)
                errs = [_rel(y, ref.detach()), _rel(xd.grad, x64.grad), _rel(wd.grad, w64.grad)]
                if has_bias:
                    errs.append(_rel(bd.grad, b64.grad))
                worst = max(worst, *errs)
    helpers.record("train_linear_fn", dict(M=M, engine=engine, worst_rel=worst, bar=LINEAR_REL))
    assert worst <= LINEAR_REL, f"LinearFn relative error {worst:.3e}"


@pytest.mark.parametrize("C", [768, 1024])
def test_layernorm_fn_vs_fp64_autograd(C):
    g = gen(1100 + C)
    worst = 0.0
    for rows in (1, 9, 320):
        ln = torch.nn.LayerNorm(C)
        torch.nn.init.normal_(ln.weight, 1.0, 0.2, generator=g)
        torch.nn.init.normal_(ln.bias, 0.0, 0.2, generator=g)
        x = torch.randn(rows, C, generator=g) * 1.7 + 0.3
        gy = torch.randn(rows, C, generator=g).double()
        lnd = torch.nn.LayerNorm(C).to(DEV)
        lnd.load_state_dict(ln.state_dict())
        xd = x.to(DEV).requires_grad_(True)
        y = A.layernorm(xd, lnd)
        y.backward(gy.float().to(DEV))
        x64 = x.double().requires_grad_(True)
        g64, b64 = (t.detach().double().requires_grad_(True) for t in (ln.weight, ln.bias))
        ref = F.layer_norm(x64, (C,), g64, b64, F32_EPS_1E5)
        ref.backward(gy)
        worst = max(worst, _rel(y, ref.detach()), _rel(xd.grad, x64.grad), _rel(lnd.weight.grad, g64.grad),
                    _rel(lnd.bias.grad, b64.grad))
    helpers.record("train_layernorm_fn", dict(C=C, worst_rel=worst, bar=LAYERNORM_FN_REL))
    assert worst <= LAYERNORM_FN_REL, f"LayerNormFn relative error {worst:.3e}"


# ------------------------------------------------------------------------------------------ EmbeddingFn / SinePosFn
def test_embedding_and_sine_pos_fns_vs_fp64_autograd():
    """y = embedding(ids) + alpha * pe: d-weight (atomics on heavily repeated ids), dx (= dy exactly) and d-alpha
    (rowdot over the pe rows, then colsum) against fp64 autograd, each within its fp32 bound."""
    g = gen(1200)
    B, T, V, D = 3, 50, 30, 96
    ids = torch.randint(0, V, (B, T), generator=g)
    ids[torch.rand(B, T, generator=g) < 0.7] = 3
    w = torch.randn(V, D, generator=g)
    alpha = torch.tensor([0.83])
    pe = R.sine_pe_table(T, D)
    gz = torch.randn(B, T, D, generator=g).double()

    wd, ad = w.to(DEV).requires_grad_(True), alpha.to(DEV).requires_grad_(True)
    y = A.EmbeddingFn.apply(ids.to(DEV), wd)
    assert torch.equal(y.detach().cpu(), w[ids]), "the forward is a gather"
    yl = y.detach().requires_grad_(True)                                         # the SinePosFn input as a leaf: dx
    z = A.SinePosFn.apply(yl, ad, pe.to(DEV))
    z.backward(gz.float().to(DEV))
    y.backward(yl.grad)

    w64, a64 = w.double().requires_grad_(True), alpha.double().requires_grad_(True)
    y64 = F.embedding(ids, w64)
    z64 = y64 + a64 * pe.double()
    z64.backward(gz)
    assert torch.equal(yl.grad.cpu(), gz.float()), "d(x + alpha pe) / dx = dy exactly"
    _within((z.detach().double().cpu() - z64.detach()).abs(), 2 * U * (y64.detach().abs() + (a64 * pe.double()).detach().abs()))
    mag = torch.zeros(V, D, dtype=torch.float64).index_add_(0, ids.reshape(-1), gz.abs().reshape(-1, D))
    n = torch.bincount(ids.reshape(-1), minlength=V).double()[:, None]
    e_w = _within((wd.grad.double().cpu() - w64.grad).abs(), n * U * mag)
    bound_a = (math.ceil(D / 32) + B * T + 10) * U * (gz * pe.double()).abs().sum()
    e_a = _within((ad.grad.double().cpu() - a64.grad).abs(), bound_a)
    helpers.record("train_embedding_sine_pos_fns", dict(dweight_err_over_bound=e_w, dalpha_err_over_bound=e_a))


# ------------------------------------------------------------------------------------------ one encoder layer, dropout on
def _mha_ref(sd, x, H, mask, keep):
    """oracle/ref_megatts2.mha with the attention dropout applied to the probabilities"""
    B, T, D = x.shape
    dh = D // H
    q, k, v = (F.linear(x, sd(f"w_{n}.weight"), sd(f"w_{n}.bias")).view(B, T, H, dh).transpose(1, 2) for n in "qkv")
    s = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(dh) + mask
    a = torch.matmul(torch.softmax(s, dim=-1) * keep, v).transpose(1, 2).reshape(B, T, D)
    return F.linear(a, sd("out_proj.0.weight"), sd("out_proj.0.bias"))


@pytest.mark.parametrize("D,H,FF", [(1024, 16, 4096), (768, 8, 1024)], ids=["plm", "adm"])
def test_encoder_layer_train_mode_dropout_vs_fp64(monkeypatch, D, H, FF):
    """TransformerEncoderLayer.forward_train with dropout 0.1 and a causal + pad mask; the three masks it draws (attention
    keep, out-projection dropout, feed-forward dropout) applied by an fp64 restatement built from the oracle's pieces."""
    from megatts2_b200.modules.transformer import TransformerEncoderLayer
    B, T, p = 2, 40, 0.1
    torch.manual_seed(1300 + D)
    layer = TransformerEncoderLayer(D, FF, conv_ff=False, n_heads=H, dropout=p)
    for ln in (layer.norm1, layer.norm2):
        torch.nn.init.normal_(ln.weight, 1.0, 0.2)
        torch.nn.init.normal_(ln.bias, 0.0, 0.2)
    sd64 = {k: v.detach().double().requires_grad_(True) for k, v in layer.state_dict().items()}
    layer = layer.to(DEV).train()
    g = gen(1301 + D)
    x = torch.randn(B, T, D, generator=g)
    gy = torch.randn(B, T, D, generator=g).double()
    lens = torch.tensor([T, T - 9], dtype=torch.int32)
    mask = make_attn_mask(lens, H, causal=True)

    dropped = []
    real_dropout = A.dropout

    def dropout(t, pp, training):
        dropped.append(t.detach().clone())
        return real_dropout(t, pp, training)
    monkeypatch.setattr(A, "dropout", dropout)
    xd = x.to(DEV).requires_grad_(True)
    with _Draws(monkeypatch) as rec:
        y = layer(xd, mask.to(DEV))
    assert [tuple(d.shape) for d in rec.draws] == [(B, H, T, T), (B, T, D), (B, T, FF)]
    keep_attn, keep_out, keep_ff = (_keep(d, p) for d in rec.draws)
    y.backward(gy.float().to(DEV))

    sd = R.SD(sd64)
    x64 = x.double().requires_grad_(True)
    h = x64 + _mha_ref(sd.sub("attn"), R.layer_norm(x64, sd("norm1.weight"), sd("norm1.bias")), H, mask.double(),
                       keep_attn) * keep_out
    z = F.linear(R.layer_norm(h, sd("norm2.weight"), sd("norm2.bias")), sd("ff.0.weight"), sd("ff.0.bias"))
    f = z * _relu_from_product(z.detach(), dropped[1]) * keep_ff
    ref = h + F.linear(f, sd("ff.3.weight"), sd("ff.3.bias"))
    ref.backward(gy)

    gmax = max(v.grad.abs().max().item() for v in sd64.values() if v.grad is not None)
    errs = {"y": _rel(y, ref.detach()), "dx": _rel(xd.grad, x64.grad)}
    for name, prm in layer.named_parameters():
        # the key bias' gradient is zero in exact arithmetic (softmax ignores a shift of a row): its error is measured
        # against 1e-3 of the layer's largest gradient
        errs[name] = _rel(prm.grad, sd64[name].grad, floor=1e-3 * gmax)
    assert len(errs) == 2 + 16
    helpers.record("train_encoder_layer", dict(D=D, bar=LAYER_REL, key_bias_bar=LAYER_KEY_BIAS, errs=errs))
    assert errs.pop("attn.w_k.bias") <= LAYER_KEY_BIAS
    assert max(errs.values()) <= LAYER_REL, {k: f"{v:.2e}" for k, v in errs.items() if v > LAYER_REL}
