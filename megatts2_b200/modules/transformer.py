"""MultiHeadAttention / TransformerEncoderLayer / TransformerEncoder with the reference's
surface (modules/transformer.py:16-57, 59-102, 105-133): same ctor kwargs, attributes,
state_dict keys (w_q/w_k/w_v, out_proj.0, norm1/2, ff.0/ff.2|ff.3, layers.{i}) and forward
signatures.  The nn.Linear / nn.Conv1d / nn.LayerNorm children only HOLD parameters; the
math runs in libmegatts2_b200 (mtts_encoder_forward_f32: LN -> packed QKV GEMM -> attention
-> out-proj + residual -> FFN, one C call for the whole stack) in eval mode.  In TRAINING mode (SURVEY.md 8f-4) the
forward is composed from megatts2_b200.autograd Functions - the same kernels plus their backward kernels, dropout
included - so ``loss.backward()`` flows through the library (linear-FF layers: the PLM / ADM trainers)."""
import copy
import ctypes as C

import torch
from torch import nn

from .. import _lib as L
from .. import autograd as A
from .. import ops, pack
from ..utils.utils import make_attn_mask


def _get_clones(module, N):
    return nn.ModuleList([copy.deepcopy(module) for _ in range(N)])


def _no_train_dropout(mod, p):
    if mod.training and p > 0:
        raise L.MttsError("training-mode dropout is outside the synthesis path (call .eval())")


class MultiHeadAttention(pack.PlanMixin, nn.Module):
    def __init__(self, qkv_dim, n_heads=8, dropout=0.):
        super().__init__()
        assert qkv_dim % n_heads == 0
        self.n_heads = n_heads
        self.head_dim = qkv_dim // n_heads
        self.dropout = dropout
        self.qkv_dim = qkv_dim
        self.w_q = nn.Linear(qkv_dim, qkv_dim, bias=True)
        self.w_k = nn.Linear(qkv_dim, qkv_dim, bias=True)
        self.w_v = nn.Linear(qkv_dim, qkv_dim, bias=True)
        self.out_proj = nn.Sequential(nn.Linear(qkv_dim, qkv_dim), nn.Dropout(dropout))
        self._plan = None

    def _packed(self):
        ps = [self.w_q.weight, self.w_q.bias, self.w_k.weight, self.w_k.bias, self.w_v.weight, self.w_v.bias,
              self.out_proj[0].weight, self.out_proj[0].bias]
        sig = pack.signature(ps)
        if self._plan is None or self._plan.sig != sig:
            pl = pack.Plan()
            pl.sig = sig
            pl.wq = pack.pack_linear(self.w_q.weight)
            pl.wkv = pack.pack_linear(pack.cat_rows(self.w_k.weight, self.w_v.weight))
            pl.bkv = pack.cat_vectors(self.w_k.bias, self.w_v.bias)
            pl.wqkv = pack.pack_qkv(self.w_q.weight, self.w_k.weight, self.w_v.weight)
            pl.bqkv = pack.cat_vectors(self.w_q.bias, self.w_k.bias, self.w_v.bias)
            pl.wo = pack.pack_linear(self.out_proj[0].weight)
            self._plan = pl
        return self._plan

    def forward(self, q, kv=None, mask=None, out=None):
        """q (B,Tq,D), kv (B,Tk,D) or None (self-attention), additive mask broadcastable to (B,H,Tq,Tk).  ``out``: an
        optional contiguous (B,Tq,D) fp32 tensor the out-projection writes into (inference only)."""
        if self.training:
            assert out is None, "training-mode attention allocates its own output"
            return self.forward_train(q, kv, mask)
        pl = self._packed()
        D = self.qkv_dim
        if kv is None:
            qkv = ops.linear(q, pl.wqkv, pl.bqkv)
            qq, kk, vv = qkv[..., :D], qkv[..., D:2 * D], qkv[..., 2 * D:]
        else:
            qq = ops.linear(q, pl.wq, self.w_q.bias.detach())
            kvp = ops.linear(kv, pl.wkv, pl.bkv)
            kk, vv = kvp[..., :D], kvp[..., D:]
        att = ops.attention(qq, kk, vv, self.n_heads, mask)
        return ops.linear(att, pl.wo, self.out_proj[0].bias.detach(), out=out)


def _mha_forward_train(self, q, kv=None, mask=None):
    """Training-mode MultiHeadAttention.forward (modules/transformer.py:35-57) on autograd Functions: three projections,
    unfused attention with dropout on the probabilities (F.scaled_dot_product_attention(..., dropout_p)), out-projection,
    nn.Dropout."""
    src = q if kv is None else kv
    qq = A.linear(q, self.w_q.weight, self.w_q.bias)
    kk = A.linear(src, self.w_k.weight, self.w_k.bias)
    vv = A.linear(src, self.w_v.weight, self.w_v.bias)
    att = A.AttentionFn.apply(qq, kk, vv, self.n_heads, mask, float(self.dropout))
    out = A.linear(att, self.out_proj[0].weight, self.out_proj[0].bias)
    return A.dropout(out, self.out_proj[1].p, True)


MultiHeadAttention.forward_train = _mha_forward_train


class TransformerEncoderLayer(pack.PlanMixin, nn.Module):
    def __init__(self, dim, ff_dim, conv_ff=False, n_heads=8, dropout=0.):
        super().__init__()
        self.dim = dim
        self.conv_ff = conv_ff
        self.n_heads = n_heads
        self.ff_dim = ff_dim
        self.p_drop = dropout
        self.norm1 = nn.LayerNorm(dim)
        self.norm2 = nn.LayerNorm(dim)
        self.attn = MultiHeadAttention(dim, n_heads=n_heads, dropout=dropout)
        self.dropout = nn.Dropout(dropout)
        if conv_ff:
            self.ff = nn.Sequential(
                nn.Conv1d(dim, ff_dim, kernel_size=5, padding=2),
                nn.ReLU(),
                nn.Conv1d(ff_dim, dim, kernel_size=5, padding=2),
            )
        else:
            self.ff = nn.Sequential(nn.Linear(dim, ff_dim), nn.ReLU(), self.dropout, nn.Linear(ff_dim, dim))
        self._plan = None

    def forward(self, x: torch.Tensor, mask: torch.Tensor = None):
        if self.training:
            return self.forward_train(x, mask)
        return run_encoder(self, [self], x, mask)

    def forward_train(self, x, mask=None):
        """Training-mode layer (modules/transformer.py:88-102), linear feed-forward: x + attn(LN1(x)); x + FF(LN2(x)) with
        FF = Linear -> ReLU -> Dropout -> Linear."""
        if self.conv_ff:
            raise L.MttsError("training through the conv feed-forward layers (MRTE phone encoder, generator trainer) is not "
                              "built yet; the PLM / ADM stacks use the linear feed-forward")
        x = x + self.attn(A.layernorm(x, self.norm1), mask=mask)
        h = A.linear(A.layernorm(x, self.norm2), self.ff[0].weight, self.ff[0].bias, relu=True)
        h = A.dropout(h, self.p_drop, True)
        return x + A.linear(h, self.ff[3].weight, self.ff[3].bias)


class TransformerEncoder(pack.PlanMixin, nn.Module):
    def __init__(self, encoder_layer: TransformerEncoderLayer, num_layers: int, norm=None):
        super().__init__()
        self.layers = _get_clones(encoder_layer, num_layers)
        self.num_layers = num_layers
        self.norm = norm
        self._plan = None

    def forward(self, x: torch.Tensor, x_lens: torch.Tensor = None, causal: bool = False) -> torch.Tensor:
        mask = make_attn_mask(x_lens, self.layers[0].n_heads, causal=causal) if x_lens is not None else None
        if self.training:
            for layer in self.layers:
                x = layer(x, mask)
            return A.layernorm(x, self.norm) if self.norm is not None else x
        y = run_encoder(self, list(self.layers), x, mask)
        if self.norm is not None:
            y = ops.layernorm(y, self.norm.weight.detach(), self.norm.bias.detach(), eps=self.norm.eps)
        return y


def encoder_plan(owner, layers):
    """Packed weights + mtts_encoder struct for a list of layers, cached on `owner`."""
    params = [p for lyr in layers for p in lyr.parameters()]
    engine = getattr(owner, "engine", None)
    engine = pack.default_engine() if engine is None else int(engine)
    sig = pack.signature(params) + (engine,)
    pl = owner._plan
    if pl is None or pl.sig != sig:
        pl = pack.Plan()
        pl.sig = sig
        l0 = layers[0]
        pl.enc = pack.build_encoder_struct(pl, layers, l0.dim, l0.n_heads, l0.ff_dim, l0.conv_ff, engine)
        owner._plan = pl
    return pl


def run_encoder(owner, layers, x, mask=None, last_row_only=False):
    for lyr in layers:
        _no_train_dropout(lyr, lyr.p_drop)
    x = ops._dev(x, name="x").contiguous()
    B, T, D = x.shape
    assert D == layers[0].dim
    pl = encoder_plan(owner, layers)
    lib = L.lib()
    y = torch.empty((B, 1, D) if last_row_only else (B, T, D), dtype=torch.float32, device=x.device)
    ws_bytes = lib.mtts_encoder_workspace_bytes(C.byref(pl.enc), B, T)
    ws = ops.workspace(ws_bytes, x.device)
    mptr, msb, msh, msq = None, 0, 0, 0
    if mask is not None:
        m = ops._dev(mask, name="mask")
        while m.dim() < 4:
            m = m.unsqueeze(0)
        m = m.expand(B, layers[0].n_heads, T, T)
        if m.stride(3) != 1 and T > 1:
            m = m.contiguous()
        mptr, msb, msh, msq = m.data_ptr(), m.stride(0), m.stride(1), m.stride(2)
    L.check(lib.mtts_encoder_forward_f32(C.byref(pl.enc), x.data_ptr(), y.data_ptr(), B, T, mptr, msb, msh, msq,
                                         int(last_row_only), ws.data_ptr(), ws.numel(), ops._stream()))
    return y
