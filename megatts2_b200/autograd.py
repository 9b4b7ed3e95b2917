"""Autograd wrappers over the C ABI (SURVEY.md 8f-4): the training-mode forwards of the drop-in modules build a graph of
these ``torch.autograd.Function``s, so ``MegaPLMTrainer`` / ``MegaADMTrainer.training_step`` (models/trainer.py:243-268,
334-355: forward under autocast, cross-entropy / L1 loss, ``loss.backward()``, AdamW) run forward AND backward through
libmegatts2_b200.  torch supplies the tape, the loss and the optimiser; every contraction, normalisation, softmax and
scatter of both passes is a hand-written kernel:

* dense layers: forward ``x W^T`` and backward ``dX = dY W``, ``dW = dY^T X`` on the wgmma tap-GEMM (bf16x3 operands
  under every tensor-core engine: the gradients are fp32-grade at any magnitude, tighter than the bf16 autocast the
  reference trains under; the fp16 planes of f16x2 would flush tiny gradients to zero) - shapes the engine does not take
  (K = 1 embeddings of the ADM, fewer than 128 rows, ragged row counts) go to the strided fp32 batched matmul;
* attention: unfused for training (the dropout inside ``F.scaled_dot_product_attention`` needs the probabilities):
  ``S = Q K^T`` -> softmax(+mask, +dropout) -> ``P V`` and the four products of its backward, all ``mtts_bmm_f32`` on head
  views given by strides (no transposes materialised);
* LayerNorm / ReLU / embedding / positional-scale backward kernels (csrc/train.cu).

Dropout masks come from torch's generator (``torch.rand``), so a training run is reproducible under ``torch.manual_seed``
but its mask stream differs from the reference's fused SDPA / nn.Dropout kernels - like any two dropout implementations.
"""
import math

import torch

from . import _lib as L
from . import ops, pack

_F32 = torch.float32
# under the trainers' ``torch.cuda.amp.autocast`` the Functions run with autocast off and fp32 inputs (the library is fp32)
_fwd = torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
_bwd = torch.amp.custom_bwd(device_type="cuda")


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


# ------------------------------------------------------------------------------------------ matmul helpers
def bmm(a, b, z1, z2, M, N, K, sa, sb, out=None, so=None, alpha=1.0, accumulate=False):
    """C[z1,z2][m,n] = alpha * sum_k A[..][m,k] B[..][k,n]; sa = (s1, s2, sm, sk), sb = (s1, s2, sk, sn), so = (s1, s2, sm, sn)
    element strides of the given base tensors."""
    if out is None:
        out = torch.empty(z1, z2, M, N, dtype=_F32, device=a.device)
        so = (z2 * M * N, M * N, N, 1)
    L.check(L.lib().mtts_bmm_f32(ops._ptr(a), *sa, ops._ptr(b), *sb, ops._ptr(out), *so, z1, z2, M, N, K, float(alpha),
                                 int(accumulate), ops._stream()))
    return out


def _tc_ok(M, K, N):
    """shapes the tensor-core tap-GEMM takes as a k = 1 layer (conv_tc_eligible in csrc/conv_tc.cu)"""
    return (pack.default_engine() != pack.ENGINE_FFMA and M >= 128 and K % 8 == 0 and K >= 32 and
            (N in (32, 64) or (N >= 128 and N % 32 == 0)) and not (K < 64 and N != 32))


def _train_fmt():
    """operand format of the training products: bf16x3 under every tensor-core engine.  Gradients span far more than the
    fp16 exponent range: an f16x2 operand below 2^-14 loses precision (|x - x^| <= 2^-22 |x| + 2^-36) and one below
    about 2^-35 becomes zero, which silently drops e.g. the weight gradient of a vocabulary row the model has learnt to
    rule out.  bf16x3 has the fp32 range, so every product is fp32-grade at any magnitude."""
    return pack.FMT_BF16X3


def matmul_nt(a, b):
    """a (M, K) @ b (N, K)^T -> (M, N), fp32-grade: tensor cores when the shape is eligible, else the fp32 batched matmul."""
    M, K = a.shape
    N = b.shape[0]
    if M == 0 or N == 0:
        return torch.zeros(M, N, dtype=_F32, device=a.device)
    if _tc_ok(M, K, N):
        fmt = _train_fmt()
        return ops.linear_tc(_c(a), pack.pack_tc_planes(_c(b), fmt))
    return bmm(a, b, 1, 1, M, N, K, (0, 0, a.stride(0), a.stride(1)), (0, 0, b.stride(1), b.stride(0)))[0, 0]


def transpose2d(x):
    """(R, C) -> contiguous (C, R) through the library's tiled copy kernel"""
    R, Cc = x.shape
    y = torch.empty(Cc, R, dtype=_F32, device=x.device)
    L.check(L.lib().mtts_copy_strided_f32(ops._ptr(x), 0, x.stride(1), x.stride(0), ops._ptr(y), 0, R, 1, 1, Cc, R, 0, ops._stream()))
    return y


def colsum(x2d, out=None, accumulate=False):
    rows, Cc = x2d.shape
    if out is None:
        out = torch.empty(Cc, dtype=_F32, device=x2d.device)
    L.check(L.lib().mtts_colsum_f32(ops._ptr(x2d), x2d.stride(0), rows, Cc, ops._ptr(out), int(accumulate), ops._stream()))
    return out


# ------------------------------------------------------------------------------------------ Functions
class LinearFn(torch.autograd.Function):
    """y = act(x W^T + b); act in {none, relu}.  x (..., K), W (N, K) as nn.Linear stores it."""

    @staticmethod
    @_fwd
    def forward(ctx, x, weight, bias, relu):
        shp = x.shape
        x2 = _c(x.reshape(-1, shp[-1]).to(_F32))
        w = weight.detach().to(_F32)
        b = bias.detach().to(_F32) if bias is not None else None
        act = L.ACT_RELU if relu else L.ACT_NONE
        M, K = x2.shape
        if _tc_ok(M, K, w.shape[0]):      # bias + activation ride in the tap-GEMM's epilogue on both engines
            y = ops.linear_tc(x2, pack.pack_tc_planes(_c(w), _train_fmt()), b, post_act=act)
        else:
            y = ops.linear(x2, pack.pack_linear(w), b, post_act=act)
        ctx.save_for_backward(x2, w, y if relu else None)
        ctx.relu, ctx.has_bias, ctx.shape = relu, bias is not None, shp
        return y.reshape(*shp[:-1], w.shape[0])

    @staticmethod
    @_bwd
    def backward(ctx, dy):
        x2, w, y = ctx.saved_tensors
        dy2 = _c(dy.reshape(-1, w.shape[0]).to(_F32))
        if ctx.relu:
            g = torch.empty_like(dy2)
            L.check(L.lib().mtts_relu_bwd_f32(ops._ptr(y), ops._ptr(dy2), ops._ptr(g), dy2.numel(), ops._stream()))
            dy2 = g
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = matmul_nt(dy2, transpose2d(w)).reshape(ctx.shape)          # dY (M,N) @ W (N,K): B operand = W^T (K,N)
        if ctx.needs_input_grad[1]:
            dw = matmul_nt(transpose2d(dy2), transpose2d(x2))               # dY^T (N,M) @ X (M,K): operands (N,M), (K,M)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = colsum(dy2)
        return dx, dw, db, None


class LayerNormFn(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, x, gamma, beta, eps):
        x2 = _c(x.reshape(-1, x.shape[-1]).to(_F32))
        g, b = gamma.detach().to(_F32), beta.detach().to(_F32)
        y = ops.layernorm(x2, g, b, eps=eps)
        ctx.save_for_backward(x2, g)
        ctx.eps, ctx.shape = eps, x.shape
        return y.reshape(x.shape)

    @staticmethod
    @_bwd
    def backward(ctx, dy):
        x2, g = ctx.saved_tensors
        rows, Cc = x2.shape
        dy2 = _c(dy.reshape(rows, Cc).to(_F32))
        dx = torch.empty_like(x2)
        nb = (rows + 7) // 8
        partial = torch.empty(nb, 2, Cc, dtype=_F32, device=x2.device)
        L.check(L.lib().mtts_layernorm_bwd_f32(ops._ptr(x2), ops._ptr(g), ops._ptr(dy2), ops._ptr(dx), ops._ptr(partial), rows, Cc,
                                               float(ctx.eps), ops._stream()))
        dgb = colsum(partial.view(nb, 2 * Cc))
        return dx.reshape(ctx.shape), dgb[:Cc], dgb[Cc:], None


class AttentionFn(torch.autograd.Function):
    """softmax(Q K^T / sqrt(dh) + mask) with dropout, times V; q (B,Tq,D), k / v (B,Tk,D), heads as strided views."""

    @staticmethod
    @_fwd
    def forward(ctx, q, k, v, n_heads, mask, p_drop):
        q, k, v = (_c(t.to(_F32)) for t in (q, k, v))
        B, Tq, D = q.shape
        Tk = k.shape[1]
        dh = D // n_heads
        H = n_heads
        scale = 1.0 / math.sqrt(dh)
        hv = lambda T: (T * D, dh, D, 1)                                      # (b, h, t, d) strides of a (B,T,D) tensor
        S = bmm(q, k, B, H, Tq, Tk, dh, hv(Tq), (Tk * D, dh, 1, D), alpha=scale)     # B operand: K^T via strides
        keep = None
        if p_drop > 0.0:
            keep = (torch.rand(B, H, Tq, Tk, device=q.device) >= p_drop).to(_F32) / (1.0 - p_drop)
        m_ptr, msb, msh, msq = None, 0, 0, 0
        if mask is not None:
            m = mask.to(_F32)
            while m.dim() < 4:
                m = m.unsqueeze(0)
            m = m.expand(B, H, Tq, Tk)
            if m.stride(3) != 1 and Tk > 1:
                m = m.contiguous()
            m_ptr, msb, msh, msq = m, m.stride(0), m.stride(1), m.stride(2)
        P = torch.empty_like(S)
        Pd = torch.empty_like(S) if keep is not None else P
        L.check(L.lib().mtts_softmax_fwd_f32(ops._ptr(S), ops._ptr(m_ptr), msb, msh, msq, B, H, Tq, Tk, ops._ptr(keep), ops._ptr(P),
                                             ops._ptr(Pd), ops._stream()))
        o = torch.empty(B, Tq, D, dtype=_F32, device=q.device)
        bmm(Pd, v, B, H, Tq, dh, Tk, (H * Tq * Tk, Tq * Tk, Tk, 1), hv(Tk)[:2] + (D, 1), out=o, so=hv(Tq))
        ctx.save_for_backward(q, k, v, P, Pd if keep is not None else None, keep)
        ctx.dims = (B, H, Tq, Tk, dh, D, scale)
        return o

    @staticmethod
    @_bwd
    def backward(ctx, do):
        q, k, v, P, Pd, keep = ctx.saved_tensors
        B, H, Tq, Tk, dh, D, scale = ctx.dims
        do = _c(do.to(_F32))
        Pd = P if Pd is None else Pd
        hv = lambda T: (T * D, dh, D, 1)
        pv = (H * Tq * Tk, Tq * Tk, Tk, 1)
        # dV[b,h] = Pd^T dO  (Tk x dh);   dPd = dO V^T  (Tq x Tk)
        dv = torch.empty_like(v)
        bmm(Pd, do, B, H, Tk, dh, Tq, (pv[0], pv[1], 1, Tk), hv(Tq)[:2] + (D, 1), out=dv, so=hv(Tk))
        dPd = bmm(do, v, B, H, Tq, Tk, dh, hv(Tq), (Tk * D, dh, 1, D))
        dS = torch.empty_like(P)
        L.check(L.lib().mtts_softmax_bwd_f32(ops._ptr(P), ops._ptr(dPd), ops._ptr(keep), ops._ptr(dS), Tk, B * H * Tq, ops._stream()))
        # dQ = scale * dS K;  dK = scale * dS^T Q
        dq = torch.empty_like(q)
        bmm(dS, k, B, H, Tq, dh, Tk, pv, hv(Tk)[:2] + (D, 1), out=dq, so=hv(Tq), alpha=scale)
        dk = torch.empty_like(k)
        bmm(dS, q, B, H, Tk, dh, Tq, (pv[0], pv[1], 1, Tk), hv(Tq)[:2] + (D, 1), out=dk, so=hv(Tk), alpha=scale)
        return dq, dk, dv, None, None, None


class EmbeddingFn(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, ids, weight):
        ids = _c(ids)
        w = weight.detach().to(_F32)
        y = ops.embed_pe(ids.reshape(1, -1), w)[0].reshape(*ids.shape, w.shape[1])
        ctx.save_for_backward(ids)
        ctx.wshape = w.shape
        return y

    @staticmethod
    @_bwd
    def backward(ctx, dy):
        (ids,) = ctx.saved_tensors
        V, D = ctx.wshape
        dy2 = _c(dy.reshape(-1, D).to(_F32))
        dw = torch.zeros(V, D, dtype=_F32, device=dy.device)
        L.check(L.lib().mtts_embedding_bwd_f32(ops._ptr(ids.reshape(-1)), ops._ptr(dy2), dy2.shape[0], D, V, ops._ptr(dw), ops._stream()))
        return None, dw


class SinePosFn(torch.autograd.Function):
    """x + alpha * pe[:T]  (SinePositionalEmbedding.forward, modules/embedding.py:94-98); alpha is a learnable scalar."""

    @staticmethod
    @_fwd
    def forward(ctx, x, alpha, pe):
        x = _c(x.to(_F32))
        y = ops.add_pe(x, pe, float(alpha.detach().reshape(-1)[0]))
        ctx.save_for_backward(pe)
        ctx.T = x.shape[1]
        return y

    @staticmethod
    @_bwd
    def backward(ctx, dy):
        (pe,) = ctx.saved_tensors
        dy2 = _c(dy.to(_F32))
        B, T, D = dy2.shape
        da = None
        if ctx.needs_input_grad[1]:
            dots = torch.empty(B * T, dtype=_F32, device=dy.device)
            L.check(L.lib().mtts_rowdot_f32(ops._ptr(dy2), ops._ptr(pe), B * T, D, T, ops._ptr(dots), ops._stream()))
            da = colsum(dots.view(B * T, 1)).reshape(1)
        return dy2, da, None


def linear(x, weight, bias=None, relu=False):
    return LinearFn.apply(x, weight, bias, relu)


def layernorm(x, ln):
    return LayerNormFn.apply(x, ln.weight, ln.bias, ln.eps)


def dropout(x, p, training):
    """nn.Dropout in training mode: mask from torch's generator, one multiply (autograd's own mul node)."""
    if not training or p <= 0.0:
        return x
    keep = (torch.rand(x.shape, device=x.device) >= p).to(x.dtype) / (1.0 - p)
    return x * keep
